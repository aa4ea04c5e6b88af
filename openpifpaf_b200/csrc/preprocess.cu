// libpifpaf_b200 -- image preprocessing on the GPU (SURVEY.md 8f rank 2).
//
// Replaces, for the inference path of the reference's Predictor (predictor.py:85-102):
//   transforms.RescaleAbsolute(long_edge, fast=True)   transforms/scale.py:154-176 -> PIL.Image.resize(BILINEAR)
//   transforms.RescaleAbsolute(long_edge, fast=False)  transforms/scale.py:60-67 -> scipy.ndimage.zoom(order=1)
//   transforms.RescaleAbsolute(long_edge, fast=True)   transforms/scale.py:41-55 -> cv2.resize(INTER_LINEAR) when
//                                                      OpenCV is importable
//   transforms.CenterPad / CenterPadTight              transforms/pad.py:15-110
// ToTensor + Normalize (transforms/__init__.py:26-33) already run inside the stem kernel (pifpaf_net_forward_u8).
//
// The reference resizes with Pillow (a third-party dependency of the reference, setup.py `pillow`; 12.2.0 in this
// image) unless OpenCV is importable.  Pillow's ImagingResample (src/libImaging/Resample.c) is restated here: a
// separable convolution, horizontal pass first into an 8-bit intermediate, then the vertical pass; coefficients are
// the antialiased triangle filter, normalised, in fixed point with 22 fractional bits (host side:
// openpifpaf_b200/preprocess.py, IEEE double arithmetic in Pillow's order), accumulated in 32-bit integers from
// 1 << 21 and shifted down -- integer arithmetic, so the resized image equals Pillow's bit for bit.
//
// The precise rescale, transforms.RescaleAbsolute(fast=False) -> scipy.ndimage.zoom(order=1) (transforms/scale.py:
// 60-67), is k_zoom_linear: one thread per canvas pixel of a whole batch, pad colour outside the window, inside it
// scipy's zoom_shift for order 1 in float64.  The per-axis taps come from the host restatement
// (preprocess.scipy_zoom_tables).  The channel axis zooms by exactly 1, so its weights are exactly 1 and 0: each of
// the four (y, x) terms is (v * wy) * wx, and the channel's zero-weight terms add +0.0, which changes nothing.  The
// sum runs in scipy's order from 0.0, and the uint8 store is scipy's: t > 0 ? t + 0.5 : 0, clamped to 255,
// truncated.  This file is built with FMA contraction on, so the arithmetic is written with __dmul_rn / __dadd_rn.
//
// The fast rescale where OpenCV is importable, cv2.resize(INTER_LINEAR) (transforms/scale.py:41-55), is
// k_resize_linear_cv, laid out like k_zoom_linear.  OpenCV resizes separably in fixed point (resize.cpp:
// resizeGeneric_, HResizeLinear into int32 rows, VResizeLinearVec_32s8u down to uint8); two taps per axis, so each
// thread recomputes the horizontal products of its two source rows in registers.  Integer arithmetic only, with
// OpenCV's int16 SIMD lanes restated in int32: the host refuses coefficients that would not fit them.  The per-axis
// taps come from the host restatement (preprocess.opencv_linear_tables), which states the coordinate rules.
#include <algorithm>
#include <cstdint>

#include "common.cuh"

namespace {

constexpr int PRECISION_BITS = 32 - 8 - 2;

__device__ __forceinline__ uint8_t clip8(int v) {
    v >>= PRECISION_BITS;
    return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal pass: src [h][w][3] -> tmp [h][tw][3]
__global__ void __launch_bounds__(256) k_resize_h(const uint8_t* __restrict__ src, int h, int w, int tw,
                                                  const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                                  uint8_t* __restrict__ tmp) {
    const long long total = (long long)h * tw;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int xx = (int)(t % tw), y = (int)(t / tw);
        const int xmin = bounds[2 * xx], xmax = bounds[2 * xx + 1];
        const int* k = kk + (size_t)xx * ksize;
        const uint8_t* row = src + ((size_t)y * w + xmin) * 3;
        int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
        for (int x = 0; x < xmax; x++) {
            const int kv = k[x];
            s0 += (int)row[3 * x] * kv; s1 += (int)row[3 * x + 1] * kv; s2 += (int)row[3 * x + 2] * kv;
        }
        uint8_t* o = tmp + ((size_t)y * tw + xx) * 3;
        o[0] = clip8(s0); o[1] = clip8(s1); o[2] = clip8(s2);
    }
}

// vertical pass: tmp [h][tw][3] -> dst rows [th] x [tw] pixels at (left, top) of a canvas with row pitch dst_pitch
__global__ void __launch_bounds__(256) k_resize_v(const uint8_t* __restrict__ tmp, int tw, int th,
                                                  const int* __restrict__ bounds, const int* __restrict__ kk, int ksize,
                                                  uint8_t* __restrict__ dst, long long dst_pitch) {
    const long long total = (long long)th * tw;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int xx = (int)(t % tw), yy = (int)(t / tw);
        const int ymin = bounds[2 * yy], ymax = bounds[2 * yy + 1];
        const int* k = kk + (size_t)yy * ksize;
        int s0 = 1 << (PRECISION_BITS - 1), s1 = s0, s2 = s0;
        for (int y = 0; y < ymax; y++) {
            const uint8_t* p = tmp + ((size_t)(y + ymin) * tw + xx) * 3;
            const int kv = k[y];
            s0 += (int)p[0] * kv; s1 += (int)p[1] * kv; s2 += (int)p[2] * kv;
        }
        uint8_t* o = dst + (size_t)yy * dst_pitch + (size_t)xx * 3;
        o[0] = clip8(s0); o[1] = clip8(s1); o[2] = clip8(s2);
    }
}

// plain copy of an image into the canvas (no rescale in that direction pair)
__global__ void __launch_bounds__(256) k_copy_rows(const uint8_t* __restrict__ src, int h, int row_bytes,
                                                   uint8_t* __restrict__ dst, long long dst_pitch) {
    const long long total = (long long)h * row_bytes;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(t % row_bytes), y = (int)(t / row_bytes);
        dst[(size_t)y * dst_pitch + x] = src[(size_t)y * row_bytes + x];
    }
}

__global__ void __launch_bounds__(256) k_fill_rgb(uint8_t* __restrict__ dst, long long n_pixels, uint8_t r, uint8_t g, uint8_t b) {
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n_pixels; t += (long long)gridDim.x * blockDim.x) {
        dst[3 * t] = r; dst[3 * t + 1] = g; dst[3 * t + 2] = b;
    }
}

// scipy's uint8 store of an interpolated value (CASE_INTERP_OUT_UINT): round half up by adding 0.5, clamp, truncate
__device__ __forceinline__ uint8_t scipy_u8(double t) {
    t = t > 0.0 ? __dadd_rn(t, 0.5) : 0.0;
    t = t > 255.0 ? 255.0 : t;
    return (uint8_t)__double2uint_rz(t);
}

// canvas [n][ch][cw][3]: one thread per pixel, each image's window at (left, top) is scipy.ndimage.zoom(order=1)
// of its source, everything else its pad colour
__global__ void __launch_bounds__(256) k_zoom_linear(const pifpaf_zoom_image_t* __restrict__ images,
                                                     const pifpaf_zoom_tap_t* __restrict__ taps,
                                                     uint8_t* __restrict__ canvas, int ch, int cw, long long total) {
    const long long plane = (long long)ch * cw;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(t / plane);
        const int p = (int)(t - (long long)b * plane);
        const pifpaf_zoom_image_t& im = images[b];
        const int yy = p / cw - im.top, xx = p % cw - im.left;
        uint8_t* o = canvas + 3 * t;
        if (yy < 0 || yy >= im.th || xx < 0 || xx >= im.tw) {
            o[0] = im.fill[0]; o[1] = im.fill[1]; o[2] = im.fill[2];
            continue;
        }
        const pifpaf_zoom_tap_t ty = taps[im.ytab + yy], tx = taps[im.xtab + xx];
        if (ty.i0 < 0 || tx.i0 < 0) {                      // mode='constant': outside the input, cval = 0
            o[0] = 0; o[1] = 0; o[2] = 0;
            continue;
        }
        const uint8_t* r0 = im.src + (size_t)ty.i0 * im.w * 3;
        const uint8_t* r1 = im.src + (size_t)ty.i1 * im.w * 3;
        const int c0 = 3 * tx.i0, c1 = 3 * tx.i1;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            double s = __dmul_rn(__dmul_rn((double)r0[c0 + c], ty.w0), tx.w0);
            s = __dadd_rn(s, __dmul_rn(__dmul_rn((double)r0[c1 + c], ty.w0), tx.w1));
            s = __dadd_rn(s, __dmul_rn(__dmul_rn((double)r1[c0 + c], ty.w1), tx.w0));
            s = __dadd_rn(s, __dmul_rn(__dmul_rn((double)r1[c1 + c], ty.w1), tx.w1));
            o[c] = scipy_u8(s);
        }
    }
}

// canvas [n][ch][cw][3]: one thread per pixel, each image's window at (left, top) is cv2.resize(INTER_LINEAR) of
// its source, everything else its pad colour
__global__ void __launch_bounds__(256) k_resize_linear_cv(const pifpaf_cv_image_t* __restrict__ images,
                                                          const pifpaf_cv_tap_t* __restrict__ taps,
                                                          uint8_t* __restrict__ canvas, int ch, int cw, long long total) {
    const long long plane = (long long)ch * cw;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(t / plane);
        const int p = (int)(t - (long long)b * plane);
        const pifpaf_cv_image_t& im = images[b];
        const int yy = p / cw - im.top, xx = p % cw - im.left;
        uint8_t* o = canvas + 3 * t;
        if (yy < 0 || yy >= im.th || xx < 0 || xx >= im.tw) {
            o[0] = im.fill[0]; o[1] = im.fill[1]; o[2] = im.fill[2];
            continue;
        }
        const pifpaf_cv_tap_t ty = taps[im.ytab + yy], tx = taps[im.xtab + xx];
        const uint8_t* r0 = im.src + ty.i0 * im.pitch;
        const uint8_t* r1 = im.src + ty.i1 * im.pitch;
        const int c0 = 3 * tx.i0, c1 = 3 * tx.i1;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            // HResizeLinear: exact int32 sums; VResizeLinearVec_32s8u: >> 4 into int16, mulhi, add, (+ 2) >> 2
            const int h0 = (int)r0[c0 + c] * tx.c0 + (int)r0[c1 + c] * tx.c1;
            const int h1 = (int)r1[c0 + c] * tx.c0 + (int)r1[c1 + c] * tx.c1;
            const int v = ((((h0 >> 4) * ty.c0) >> 16) + (((h1 >> 4) * ty.c1) >> 16) + 2) >> 2;
            o[c] = (uint8_t)(v > 255 ? 255 : v);
        }
    }
}

inline int grid_for(long long total) { return (int)std::min<long long>((total + 255) / 256, 132LL * 16); }

// the taps of one axis of one image lie within the staged table and index its source
bool taps_ok(const pifpaf_zoom_tap_t* taps, int64_t n_taps, int64_t first, int32_t n_out, int32_t n_in) {
    if (first < 0 || first + n_out > n_taps) return false;
    for (int32_t k = 0; k < n_out; k++) {
        const pifpaf_zoom_tap_t& tp = taps[first + k];
        if (tp.i0 == -1) continue;
        if (tp.i0 < 0 || tp.i0 >= n_in || tp.i1 < 0 || tp.i1 >= n_in) return false;
    }
    return true;
}

// the taps of one axis of one image lie within the staged table, index its source, and keep OpenCV's int16 lanes
// from saturating: coefficients >= 0 summing to at most 2048, so (H >> 4) <= 255 * 2048 >> 4 < 2^15
bool cv_taps_ok(const pifpaf_cv_tap_t* taps, int64_t n_taps, int64_t first, int32_t n_out, int32_t n_in) {
    if (first < 0 || first + n_out > n_taps) return false;
    for (int32_t k = 0; k < n_out; k++) {
        const pifpaf_cv_tap_t& tp = taps[first + k];
        if (tp.i0 < 0 || tp.i0 >= n_in || tp.i1 < 0 || tp.i1 >= n_in) return false;
        if (tp.c0 < 0 || tp.c1 < 0 || tp.c0 + tp.c1 > 2048) return false;
    }
    return true;
}

}  // namespace

extern "C" {

int pifpaf_image_fill_rgb(uint8_t* dst_dev, int64_t n_pixels, int32_t r, int32_t g, int32_t b, void* stream_v) {
    PIFPAF_CHECK_ARG(dst_dev != nullptr && n_pixels >= 0, "bad fill arguments");
    PIFPAF_CHECK_ARG(r >= 0 && r <= 255 && g >= 0 && g <= 255 && b >= 0 && b <= 255, "fill colour out of range");
    if (n_pixels == 0) return PIFPAF_OK;
    k_fill_rgb<<<grid_for(n_pixels), 256, 0, reinterpret_cast<cudaStream_t>(stream_v)>>>(dst_dev, n_pixels, (uint8_t)r, (uint8_t)g, (uint8_t)b);
    PIFPAF_LAUNCH_CHECK();
    return PIFPAF_OK;
}

int pifpaf_image_resize_bilinear_u8(const uint8_t* src_dev, int32_t src_h, int32_t src_w,
                                    uint8_t* dst_dev, int64_t dst_pitch_bytes, int32_t dst_h, int32_t dst_w,
                                    const int32_t* xbounds_dev, const int32_t* xkk_dev, int32_t xksize,
                                    const int32_t* ybounds_dev, const int32_t* ykk_dev, int32_t yksize,
                                    uint8_t* tmp_dev, void* stream_v) {
    PIFPAF_CHECK_ARG(src_dev != nullptr && dst_dev != nullptr, "image pointer is null");
    PIFPAF_CHECK_ARG(src_h >= 1 && src_w >= 1 && dst_h >= 1 && dst_w >= 1, "bad image size");
    PIFPAF_CHECK_ARG(dst_pitch_bytes >= (int64_t)dst_w * 3, "destination pitch too small");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    const bool need_h = dst_w != src_w, need_v = dst_h != src_h;          // Resample.c: ImagingResample
    PIFPAF_CHECK_ARG(!need_h || (xbounds_dev && xkk_dev && xksize >= 1), "horizontal coefficients missing");
    PIFPAF_CHECK_ARG(!need_v || (ybounds_dev && ykk_dev && yksize >= 1), "vertical coefficients missing");
    PIFPAF_CHECK_ARG(!(need_h && need_v) || tmp_dev != nullptr, "intermediate buffer [src_h][dst_w][3] missing");
    if (need_h && need_v) {
        k_resize_h<<<grid_for((long long)src_h * dst_w), 256, 0, st>>>(src_dev, src_h, src_w, dst_w, xbounds_dev, xkk_dev, xksize, tmp_dev);
        PIFPAF_LAUNCH_CHECK();
        k_resize_v<<<grid_for((long long)dst_h * dst_w), 256, 0, st>>>(tmp_dev, dst_w, dst_h, ybounds_dev, ykk_dev, yksize, dst_dev, dst_pitch_bytes);
        PIFPAF_LAUNCH_CHECK();
    } else if (need_h) {
        // rows go straight to the canvas: the "intermediate" is the destination (pitch handled by a per-row launch
        // shape: tmp layout [h][tw][3] only matches a dense destination, so resize into tmp when the pitch differs)
        if (dst_pitch_bytes == (int64_t)dst_w * 3) {
            k_resize_h<<<grid_for((long long)src_h * dst_w), 256, 0, st>>>(src_dev, src_h, src_w, dst_w, xbounds_dev, xkk_dev, xksize, dst_dev);
            PIFPAF_LAUNCH_CHECK();
        } else {
            PIFPAF_CHECK_ARG(tmp_dev != nullptr, "intermediate buffer missing");
            k_resize_h<<<grid_for((long long)src_h * dst_w), 256, 0, st>>>(src_dev, src_h, src_w, dst_w, xbounds_dev, xkk_dev, xksize, tmp_dev);
            PIFPAF_LAUNCH_CHECK();
            k_copy_rows<<<grid_for((long long)dst_h * dst_w * 3), 256, 0, st>>>(tmp_dev, dst_h, dst_w * 3, dst_dev, dst_pitch_bytes);
            PIFPAF_LAUNCH_CHECK();
        }
    } else if (need_v) {
        k_resize_v<<<grid_for((long long)dst_h * dst_w), 256, 0, st>>>(src_dev, dst_w, dst_h, ybounds_dev, ykk_dev, yksize, dst_dev, dst_pitch_bytes);
        PIFPAF_LAUNCH_CHECK();
    } else {
        k_copy_rows<<<grid_for((long long)dst_h * dst_w * 3), 256, 0, st>>>(src_dev, dst_h, dst_w * 3, dst_dev, dst_pitch_bytes);
        PIFPAF_LAUNCH_CHECK();
    }
    return PIFPAF_OK;
}

int pifpaf_image_zoom_linear_u8(const pifpaf_zoom_image_t* images, int32_t n_images,
                                const pifpaf_zoom_tap_t* taps, int64_t n_taps,
                                void* workspace_dev, int64_t workspace_bytes,
                                uint8_t* canvas_dev, int32_t canvas_h, int32_t canvas_w, void* stream_v) {
    PIFPAF_CHECK_ARG(images != nullptr && n_images >= 1, "no images");
    PIFPAF_CHECK_ARG(taps != nullptr && n_taps >= 1, "tap tables missing");
    PIFPAF_CHECK_ARG(canvas_dev != nullptr && workspace_dev != nullptr, "canvas or workspace pointer is null");
    PIFPAF_CHECK_ARG(canvas_h >= 1 && canvas_w >= 1, "bad canvas size");
    const size_t desc_bytes = sizeof(pifpaf_zoom_image_t) * (size_t)n_images;
    const size_t tap_bytes = sizeof(pifpaf_zoom_tap_t) * (size_t)n_taps;
    PIFPAF_CHECK_ARG(workspace_bytes >= 0 && (size_t)workspace_bytes >= desc_bytes + tap_bytes, "workspace too small");
    for (int32_t i = 0; i < n_images; i++) {
        const pifpaf_zoom_image_t& im = images[i];
        PIFPAF_CHECK_ARG(im.src != nullptr, "image pointer is null");
        PIFPAF_CHECK_ARG(im.h >= 1 && im.w >= 1 && im.th >= 1 && im.tw >= 1, "bad image size");
        PIFPAF_CHECK_ARG(im.left >= 0 && im.top >= 0 && (int64_t)im.left + im.tw <= canvas_w
                         && (int64_t)im.top + im.th <= canvas_h, "window outside the canvas");
        PIFPAF_CHECK_ARG(taps_ok(taps, n_taps, im.ytab, im.th, im.h), "row taps missing or outside the source");
        PIFPAF_CHECK_ARG(taps_ok(taps, n_taps, im.xtab, im.tw, im.w), "column taps missing or outside the source");
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    auto* ws = static_cast<uint8_t*>(workspace_dev);
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(ws, images, desc_bytes, cudaMemcpyHostToDevice, st));
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(ws + desc_bytes, taps, tap_bytes, cudaMemcpyHostToDevice, st));
    const long long total = (long long)n_images * canvas_h * canvas_w;
    k_zoom_linear<<<grid_for(total), 256, 0, st>>>(reinterpret_cast<const pifpaf_zoom_image_t*>(ws),
                                                   reinterpret_cast<const pifpaf_zoom_tap_t*>(ws + desc_bytes),
                                                   canvas_dev, canvas_h, canvas_w, total);
    PIFPAF_LAUNCH_CHECK();
    return PIFPAF_OK;
}

int pifpaf_image_resize_linear_cv_u8(const pifpaf_cv_image_t* images, int32_t n_images,
                                     const pifpaf_cv_tap_t* taps, int64_t n_taps,
                                     void* workspace_dev, int64_t workspace_bytes,
                                     uint8_t* canvas_dev, int32_t canvas_h, int32_t canvas_w, void* stream_v) {
    PIFPAF_CHECK_ARG(images != nullptr && n_images >= 1, "no images");
    PIFPAF_CHECK_ARG(taps != nullptr && n_taps >= 1, "tap tables missing");
    PIFPAF_CHECK_ARG(canvas_dev != nullptr && workspace_dev != nullptr, "canvas or workspace pointer is null");
    PIFPAF_CHECK_ARG(canvas_h >= 1 && canvas_w >= 1, "bad canvas size");
    const size_t desc_bytes = sizeof(pifpaf_cv_image_t) * (size_t)n_images;
    const size_t tap_bytes = sizeof(pifpaf_cv_tap_t) * (size_t)n_taps;
    PIFPAF_CHECK_ARG(workspace_bytes >= 0 && (size_t)workspace_bytes >= desc_bytes + tap_bytes, "workspace too small");
    for (int32_t i = 0; i < n_images; i++) {
        const pifpaf_cv_image_t& im = images[i];
        PIFPAF_CHECK_ARG(im.src != nullptr, "image pointer is null");
        PIFPAF_CHECK_ARG(im.h >= 1 && im.w >= 1 && im.th >= 1 && im.tw >= 1, "bad image size");
        PIFPAF_CHECK_ARG(im.pitch >= 3 * (int64_t)im.w, "source pitch too small");
        PIFPAF_CHECK_ARG(im.left >= 0 && im.top >= 0 && (int64_t)im.left + im.tw <= canvas_w
                         && (int64_t)im.top + im.th <= canvas_h, "window outside the canvas");
        PIFPAF_CHECK_ARG(cv_taps_ok(taps, n_taps, im.ytab, im.th, im.h), "row taps missing, outside the source or "
                         "with coefficients outside [0, 2048]");
        PIFPAF_CHECK_ARG(cv_taps_ok(taps, n_taps, im.xtab, im.tw, im.w), "column taps missing, outside the source or "
                         "with coefficients outside [0, 2048]");
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    auto* ws = static_cast<uint8_t*>(workspace_dev);
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(ws, images, desc_bytes, cudaMemcpyHostToDevice, st));
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(ws + desc_bytes, taps, tap_bytes, cudaMemcpyHostToDevice, st));
    const long long total = (long long)n_images * canvas_h * canvas_w;
    k_resize_linear_cv<<<grid_for(total), 256, 0, st>>>(reinterpret_cast<const pifpaf_cv_image_t*>(ws),
                                                        reinterpret_cast<const pifpaf_cv_tap_t*>(ws + desc_bytes),
                                                        canvas_dev, canvas_h, canvas_w, total);
    PIFPAF_LAUNCH_CHECK();
    return PIFPAF_OK;
}

}  // extern "C"
