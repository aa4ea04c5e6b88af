// libpifpaf_b200 -- CifCaf decoder for sm_90a.
//
// H100-native re-design of the reference's CPU decoder (paths relative to
// the reference's src/openpifpaf/csrc/):
//   CifHr::accumulate/add_gauss   src/cif_hr.cpp:28-89      -> k_cif_compact + k_cifhr_tiles
//   CifSeeds::fill/get            src/cif_seeds.cpp:33-114  -> k_seed_candidates + k_seed_sort
//   CafScored::fill               src/caf_scored.cpp:29-83  -> k_caf_scored
//   CifCaf::call_* / _grow / ...  src/cifcaf.cpp:126-449    -> k_grow (+ k_force_complete)
//   Occupancy                     src/occupancy.cpp:13-77   -> byte map with epoch tags
//   NMSKeypoints::call            src/nms_keypoints.cpp:17-69 -> k_nms, k_pack
//
// Design (see DESIGN.md): images are independent, so every kernel is batched over
// the image index; the order-dependent float accumulation of CifHr is turned from
// a scatter into a per-pixel GATHER over an order-preserving compacted cell list so
// that the result is bit-identical to the sequential reference; the frontier
// priority queue is the libstdc++ binary heap restated in shared memory (same tie
// order) driven by one thread, while the CAF list scans behind every frontier
// entry are evaluated eagerly by one warp each.
//
// This translation unit is compiled with -fmad=false: the reference arithmetic
// has no fused multiply-adds and parity needs the same roundings.
#include <algorithm>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "common.cuh"

namespace {

constexpr int NT = 256;            // threads per CTA for the streaming kernels
constexpr int NW = NT / 32;
constexpr int SORT_NT = 1024;
constexpr int TILE = 32;           // CifHr tile edge in hi-res pixels
constexpr int LIST_SMEM_ENTRIES = 8192;   // CAF list entries (c,x,y) staged in shared memory per image (96 KB)

struct Dims {
    int B, F, C, K;
    int h, w, hw;
    int cif_stride, caf_stride;
    int H, W, Wp;        // hi-res map size and padded row pitch (floats)
    int Ho, Wo;          // occupancy map size
    int tiles_x, tiles_y;
    int max_ann;
};

struct GrowParams {
    double keypoint_threshold, keypoint_threshold_rel;
    int reverse_match, greedy;
    double occ_reduction, occ_min_scale_reduced;
    double nms_suppression, nms_instance_threshold, nms_keypoint_threshold;
    float defer_radius;      // k_grow: a seed within defer_radius * scale of a seed picked in the same round waits
};

// ---------------------------------------------------------------------------
// order-preserving block compaction of up to two flags per thread.
// Every thread of the CTA must call it.  base0/base1 are CTA-uniform running
// totals held in registers.  wc is shared scratch of NWARPS ints.
template <int NWARPS>
__device__ __forceinline__ void block_compact2(bool f0, bool f1, int& base0, int& base1,
                                               int& pos0, int& pos1, int* wc) {
    const unsigned m0 = __ballot_sync(0xffffffffu, f0);
    const unsigned m1 = __ballot_sync(0xffffffffu, f1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) wc[warp] = __popc(m0) | (__popc(m1) << 16);
    __syncthreads();
    int off0 = 0, off1 = 0, tot0 = 0, tot1 = 0;
#pragma unroll
    for (int w2 = 0; w2 < NWARPS; w2++) {
        const int c = wc[w2];
        const int c0 = c & 0xffff, c1 = c >> 16;
        if (w2 < warp) { off0 += c0; off1 += c1; }
        tot0 += c0; tot1 += c1;
    }
    const unsigned lt = (1u << lane) - 1u;
    pos0 = base0 + off0 + __popc(m0 & lt);
    pos1 = base1 + off1 + __popc(m1 & lt);
    base0 += tot0;
    base1 += tot1;
    __syncthreads();
}

__device__ __forceinline__ long long clamp_ll(long long v, long long lo, long long hi) {
    return v < lo ? lo : (hi < v ? hi : v);
}

// src/cif_hr.cpp:18-25
__device__ __forceinline__ float approx_exp(float x) {
    if ((double)x > 2.0 || (double)x < -2.0) return 0.0f;
    x = (float)(1.0 + (double)x / 8.0);
    x = x * x;
    x = x * x;
    x = x * x;
    return x;
}

// The CifHr map is SPARSE: only 32x32 tiles touched by a contributing cell are ever written; a tile is
// valid for this call iff its epoch tag equals the call's epoch, otherwise every pixel of it reads as the
// never-written 0.0 of a fresh reference buffer (src/cif_hr.cpp:97-114).
struct HrView {
    const float* hr;              // image base [F][H][Wp]
    const unsigned* tile_epoch;   // image base [F][tiles]
    unsigned epoch;
    int F, H, W, Wp, tiles_x, tiles;
};

// src/cif_seeds.cpp:17-30 == src/caf_scored.cpp:15-26.
__device__ __forceinline__ float cifhr_value(const HrView& v, double revision, long long f, float x, float y,
                                             float default_value) {
    const float max_x = (float)((double)(float)v.W - 0.51);
    const float max_y = (float)((double)(float)v.H - 0.51);
    if (f >= v.F || (double)x < -0.49 || (double)y < -0.49 || x > max_x || y > max_y) return default_value;
    const long long yi = (long long)((double)y + 0.5), xi = (long long)((double)x + 0.5);
    const int tile = (int)(yi / TILE) * v.tiles_x + (int)(xi / TILE);
    float stored = 0.0f;
    if (v.tile_epoch[(size_t)f * v.tiles + tile] == v.epoch) stored = v.hr[((size_t)f * v.H + yi) * v.Wp + xi];
    const float value = (float)((double)stored - revision);
    if ((double)value < 0.0) return default_value;
    return value;
}

// ---------------------------------------------------------------------------
// CifHr step 1: compact the cells that contribute (src/cif_hr.cpp:36-51), in
// (j,i) order, with their add_gauss box (src/cif_hr.cpp:61-64).
// det != 0: CifDetHr::accumulate (src/cif_hr.cpp:124-150) on a [F][6][h][w] field -- width / height at components
// 4 / 5, both tested against min_scale, sigma = max(1, 0.1 * min(w, h) * stride).
__global__ void __launch_bounds__(NT) k_cif_compact(const float* __restrict__ cif, Dims d, int det,
                                                    double threshold, long long neighbors,
                                                    float min_scale_f, double factor,
                                                    float4* __restrict__ cells, int4* __restrict__ boxes,
                                                    int* __restrict__ counts,
                                                    unsigned* __restrict__ tile_epoch, unsigned epoch,
                                                    int* __restrict__ worklist, int* __restrict__ work_count) {
    __shared__ int wc[NW];
    const int f = blockIdx.x, b = blockIdx.y;
    const float* cf = cif + ((size_t)(b * d.F + f) * (det ? 6 : 5)) * d.hw;
    float4* out_c = cells + (size_t)(b * d.F + f) * d.hw;
    int4* out_b = boxes + (size_t)(b * d.F + f) * d.hw;
    int base = 0, dummy = 0;
    for (int start = 0; start < d.hw; start += NT) {
        const int idx = start + threadIdx.x;
        bool flag = false;
        float v = 0.f, scale = 0.f;
        if (idx < d.hw) {
            v = cf[1 * d.hw + idx];
            if (!((double)v < threshold)) {
                scale = cf[4 * d.hw + idx];
                if (!(scale < min_scale_f)) flag = true;
                if (det) {
                    const float bh = cf[5 * d.hw + idx];
                    if (bh < min_scale_f) flag = false;
                    scale = fminf(scale, bh);
                }
            }
        }
        int pos, pos1;
        block_compact2<NW>(flag, false, base, dummy, pos, pos1, wc);
        if (flag) {
            const float x = cf[2 * d.hw + idx] * (float)d.cif_stride;
            const float y = cf[3 * d.hw + idx] * (float)d.cif_stride;
            const float sigma = fmaxf(1.0f, (float)((det ? 0.1 : 0.5) * (double)scale * (double)d.cif_stride));
            const float vn = (float)((double)(v / (float)neighbors) * factor);
            const float truncate = 1.0f;
            const long long minx = clamp_ll((long long)(x - truncate * sigma), 0, d.W - 1);
            const long long miny = clamp_ll((long long)(y - truncate * sigma), 0, d.H - 1);
            const long long maxx = clamp_ll((long long)(x + truncate * sigma + 1.0f), minx + 1, d.W);
            const long long maxy = clamp_ll((long long)(y + truncate * sigma + 1.0f), miny + 1, d.H);
            out_c[pos] = make_float4(x, y, sigma, vn);
            out_b[pos] = make_int4((int)minx, (int)miny, (int)maxx, (int)maxy);
            // first toucher of a tile in this call appends it to the worklist
            const int tiles = d.tiles_x * d.tiles_y;
            for (int ty = (int)miny / TILE; ty <= ((int)maxy - 1) / TILE; ty++)
                for (int tx = (int)minx / TILE; tx <= ((int)maxx - 1) / TILE; tx++) {
                    const int gid = (b * d.F + f) * tiles + ty * d.tiles_x + tx;
                    if (atomicExch(&tile_epoch[gid], epoch) != epoch) worklist[atomicAdd(work_count, 1)] = gid;
                }
        }
    }
    if (threadIdx.x == 0) counts[b * d.F + f] = base;
}

// CifHr step 2: one CTA per 32x32 hi-res tile gathers, in cell order, every
// compacted cell whose box touches the tile (src/cif_hr.cpp:66-88 per pixel).
// Fuses the clear: each pixel is written exactly once and never read.
__global__ void __launch_bounds__(NT) k_cifhr_tiles(Dims d, double revision,
                                                    const float4* __restrict__ cells,
                                                    const int4* __restrict__ boxes,
                                                    const int* __restrict__ counts,
                                                    const int* __restrict__ worklist,
                                                    const int* __restrict__ work_count,
                                                    float* __restrict__ cifhr) {
    __shared__ int wc[NW];
    __shared__ float4 s_cell[NT];
    __shared__ int4 s_box[NT];
    const int n_work = *work_count;
    const int tiles = d.tiles_x * d.tiles_y;
    for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
    const int gid = worklist[wi];
    const int tile = gid % tiles, bf = gid / tiles;
    const int f = bf % d.F, b = bf / d.F;
    const int tx0 = (tile % d.tiles_x) * TILE, ty0 = (tile / d.tiles_x) * TILE;
    const int px = tx0 + (threadIdx.x & 7) * 4;
    const int py = ty0 + (threadIdx.x >> 3);
    const float4* in_c = cells + (size_t)(b * d.F + f) * d.hw;
    const int4* in_b = boxes + (size_t)(b * d.F + f) * d.hw;
    const int n = counts[b * d.F + f];
    const float rev_f = (float)revision;
    const float rev_p1_f = (float)(revision + 1.0);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};

    for (int start = 0; start < n; start += NT) {
        const int e = start + threadIdx.x;
        bool flag = false;
        float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
        int4 bx = make_int4(0, 0, 0, 0);
        if (e < n) {
            bx = in_b[e];
            flag = bx.x < tx0 + TILE && bx.z > tx0 && bx.y < ty0 + TILE && bx.w > ty0;
            if (flag) c = in_c[e];
        }
        int m = 0, dummy = 0, pos, pos1;
        block_compact2<NW>(flag, false, m, dummy, pos, pos1, wc);
        if (flag) { s_cell[pos] = c; s_box[pos] = bx; }
        __syncthreads();
        for (int k = 0; k < m; k++) {
            const float4 cc = s_cell[k];
            const int4 bb = s_box[k];
            if (py < bb.y || py >= bb.w) continue;
            const float sigma2 = cc.z * cc.z;           // truncate^2 * sigma2 == sigma2 for truncate 1
            const float dyf = (float)py - cc.y;
            const float deltay2 = dyf * dyf;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int xx = px + q;
                if (xx < bb.x || xx >= bb.z) continue;
                const float dxf = (float)xx - cc.x;
                const float deltax2 = dxf * dxf;
                if (deltax2 + deltay2 > sigma2) continue;
                float vv;
                if ((double)deltax2 < 0.25 && (double)deltay2 < 0.25) {
                    vv = cc.w;
                } else {
                    vv = cc.w * approx_exp((float)(-0.5 * (double)(deltax2 + deltay2) / (double)sigma2));
                }
                float entry = fmaxf(acc[q], rev_f) + vv;
                acc[q] = fminf(entry, rev_p1_f);
            }
        }
        __syncthreads();
    }
    if (py < d.H) {
        float4* dst = reinterpret_cast<float4*>(cifhr + ((size_t)(b * d.F + f) * d.H + py) * d.Wp + px);
        *dst = make_float4(acc[0], acc[1], acc[2], acc[3]);
    }
    }   // worklist loop
}

// get_cifhr()/tap support: make image b's map dense by zero-filling the tiles not written in this call.
__global__ void __launch_bounds__(NT) k_cifhr_materialize(Dims d, int b, unsigned* __restrict__ tile_epoch,
                                                          unsigned epoch, float* __restrict__ cifhr) {
    const int tile = blockIdx.x, f = blockIdx.y;
    const int tiles = d.tiles_x * d.tiles_y;
    const size_t gid = (size_t)(b * d.F + f) * tiles + tile;
    if (tile_epoch[gid] == epoch) return;
    const int px = (tile % d.tiles_x) * TILE + (threadIdx.x & 7) * 4;
    const int py = (tile / d.tiles_x) * TILE + (threadIdx.x >> 3);
    if (py < d.H)
        *reinterpret_cast<float4*>(cifhr + ((size_t)(b * d.F + f) * d.H + py) * d.Wp + px) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    if (threadIdx.x == 0) tile_epoch[gid] = epoch;
}

// ---------------------------------------------------------------------------
// CifSeeds::fill (src/cif_seeds.cpp:33-66), per (image, field), order preserving.
__global__ void __launch_bounds__(NT) k_seed_candidates(const float* __restrict__ cif, Dims d,
                                                        const float* __restrict__ cifhr,
                                                        const unsigned* __restrict__ tile_epoch, unsigned epoch,
                                                        double revision,
                                                        double threshold, int ablation_nms, int no_rescore, int det,
                                                        float* __restrict__ seg_v, float4* __restrict__ seg_xys,
                                                        int* __restrict__ seg_counts) {
    // det != 0: CifDetSeeds::fill (src/cif_seeds.cpp:69-90) on a [F][6][h][w] field; seg_xys = (x, y, w, h)
    __shared__ int wc[NW];
    const int f = blockIdx.x, b = blockIdx.y;
    const float* cf = cif + ((size_t)(b * d.F + f) * (det ? 6 : 5)) * d.hw;
    HrView hv;
    hv.hr = cifhr + (size_t)b * d.F * d.H * d.Wp;
    hv.tiles_x = d.tiles_x; hv.tiles = d.tiles_x * d.tiles_y;
    hv.tile_epoch = tile_epoch + (size_t)b * d.F * hv.tiles; hv.epoch = epoch;
    hv.F = d.F; hv.H = d.H; hv.W = d.W; hv.Wp = d.Wp;
    float* out_v = seg_v + (size_t)(b * d.F + f) * d.hw;
    float4* out_x = seg_xys + (size_t)(b * d.F + f) * d.hw;
    int base = 0, dummy = 0;
    for (int start = 0; start < d.hw; start += NT) {
        const int idx = start + threadIdx.x;
        bool flag = false;
        float c = 0.f, x = 0.f, y = 0.f;
        if (idx < d.hw) {
            c = cf[1 * d.hw + idx];
            flag = !((double)c < threshold);
            if (flag && ablation_nms) {
                // torch.max_pool2d(confidence, 3, 1, 1): src/cif_seeds.cpp:36-40,49-51
                const int j = idx / d.w, i = idx % d.w;
                float m = c;
                for (int dj = -1; dj <= 1; dj++)
                    for (int di = -1; di <= 1; di++) {
                        const int jj = j + dj, ii = i + di;
                        if (jj < 0 || jj >= d.h || ii < 0 || ii >= d.w) continue;
                        m = fmaxf(m, cf[1 * d.hw + jj * d.w + ii]);
                    }
                if (c < m) flag = false;
            }
            if (flag) {
                x = cf[2 * d.hw + idx] * (float)d.cif_stride;
                y = cf[3 * d.hw + idx] * (float)d.cif_stride;
                if (!no_rescore) {
                    const float hval = cifhr_value(hv, revision, f, x, y, -1.0f);
                    c = (float)(0.9 * (double)hval + 0.1 * (double)c);
                }
                flag = !((double)c < threshold);
            }
        }
        int pos, pos1;
        block_compact2<NW>(flag, false, base, dummy, pos, pos1, wc);
        if (flag) {
            const float s = cf[4 * d.hw + idx] * (float)d.cif_stride;
            out_v[pos] = c;
            out_x[pos] = make_float4(x, y, s, det ? cf[5 * d.hw + idx] * (float)d.cif_stride : 0.f);
        }
    }
    if (threadIdx.x == 0) seg_counts[b * d.F + f] = base;
}

__device__ __forceinline__ unsigned float_key_desc(float v) {
    const unsigned bits = __float_as_uint(v);
    const unsigned asc = bits ^ ((bits >> 31) ? 0xffffffffu : 0x80000000u);
    return ~asc;   // ascending key order == descending v
}

// CifSeeds::get (src/cif_seeds.cpp:93-114): sort by v descending.  One CTA per
// image: concatenate the per-field segments (fill order) and run a stable LSD
// radix sort, so exact float ties keep fill order (f, j, i) -- std::sort in the
// reference leaves tie order unspecified.
__global__ void __launch_bounds__(SORT_NT) k_seed_sort(Dims d, const int* __restrict__ seg_counts,
                                                       const float* __restrict__ seg_v,
                                                       const float4* __restrict__ seg_xys,
                                                       unsigned* __restrict__ keys_a, unsigned* __restrict__ vals_a,
                                                       unsigned* __restrict__ keys_b, unsigned* __restrict__ vals_b,
                                                       int* __restrict__ seed_f, float4* __restrict__ seed_vxys,
                                                       float* __restrict__ seed_extra,     // DetSeed::h, or null
                                                       int* __restrict__ n_seeds) {
    extern __shared__ unsigned char smem_raw[];
    int* s_off = reinterpret_cast<int*>(smem_raw);                 // F + 1
    int* hist = s_off + ((d.F + 1 + 3) & ~3);                      // 256
    int* dbase = hist + 256;                                       // 256
    int* wsum = dbase + 256;                                       // 8
    unsigned short* wc = reinterpret_cast<unsigned short*>(wsum + 8);   // 32 x 256
    __shared__ int s_skip;

    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t img = (size_t)b * d.F * d.hw;
    const float* in_v = seg_v + img;
    const float4* in_x = seg_xys + img;
    unsigned* kin = keys_a + img; unsigned* vin = vals_a + img;
    unsigned* kout = keys_b + img; unsigned* vout = vals_b + img;

    if (tid == 0) {
        int run = 0;
        for (int f = 0; f < d.F; f++) { s_off[f] = run; run += seg_counts[b * d.F + f]; }
        s_off[d.F] = run;
    }
    __syncthreads();
    const int n = s_off[d.F];
    for (int f = 0; f < d.F; f++) {
        const int off = s_off[f], cnt = s_off[f + 1] - off;
        for (int p = tid; p < cnt; p += SORT_NT) {
            const unsigned src = (unsigned)(f * d.hw + p);
            kin[off + p] = float_key_desc(in_v[src]);
            vin[off + p] = src;
        }
    }
    __syncthreads();

    for (int pass = 0; pass < 4; pass++) {
        const int shift = pass * 8;
        if (tid < 256) hist[tid] = 0;
        if (tid == 0) s_skip = 0;
        __syncthreads();
        for (int i = tid; i < n; i += SORT_NT) atomicAdd(&hist[(kin[i] >> shift) & 255u], 1);
        __syncthreads();
        if (tid < 256 && n > 0 && hist[tid] == n) s_skip = 1;
        __syncthreads();
        const int skip = s_skip;
        __syncthreads();
        if (skip || n == 0) continue;       // CTA-uniform
        int excl_local = 0;
        if (tid < 256) {
            const int v = hist[tid];
            int incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            if (lane == 31) wsum[warp] = incl;
            excl_local = incl - v;
        }
        __syncthreads();
        if (tid < 256) {
            int add = 0;
            for (int w2 = 0; w2 < warp; w2++) add += wsum[w2];
            dbase[tid] = excl_local + add;
        }
        __syncthreads();
        for (int t0 = 0; t0 < n; t0 += SORT_NT) {
#pragma unroll
            for (int q = 0; q < 4; q++) reinterpret_cast<unsigned*>(wc)[tid + q * SORT_NT] = 0u;
            __syncthreads();
            const int i = t0 + tid;
            const bool valid = i < n;
            const unsigned key = valid ? kin[i] : 0u;
            const unsigned dg = valid ? ((key >> shift) & 255u) : 256u;
            const unsigned peers = __match_any_sync(0xffffffffu, dg);
            const int rank = __popc(peers & ((1u << lane) - 1u));
            if (valid && rank == 0) wc[warp * 256 + dg] = (unsigned short)__popc(peers);
            __syncthreads();
            int tile_tot = 0;
            if (tid < 256) {
                int run = 0;
                for (int w2 = 0; w2 < 32; w2++) {
                    const int c = wc[w2 * 256 + tid];
                    wc[w2 * 256 + tid] = (unsigned short)run;
                    run += c;
                }
                tile_tot = run;
            }
            __syncthreads();
            if (valid) {
                const int dst = dbase[dg] + wc[warp * 256 + dg] + rank;
                kout[dst] = key;
                vout[dst] = vin[i];
            }
            __syncthreads();
            if (tid < 256) dbase[tid] += tile_tot;
        }
        __syncthreads();
        unsigned* t;
        t = kin; kin = kout; kout = t;
        t = vin; vin = vout; vout = t;
    }
    __syncthreads();
    for (int i = tid; i < n; i += SORT_NT) {
        const unsigned src = vin[i];
        const float4 xs = in_x[src];
        seed_f[img + i] = (int)(src / (unsigned)d.hw);
        seed_vxys[img + i] = make_float4(in_v[src], xs.x, xs.y, xs.z);
        if (seed_extra != nullptr) seed_extra[img + i] = xs.w;
    }
    if (tid == 0) n_seeds[b] = n;
}

// ---------------------------------------------------------------------------
// CafScored::fill (src/caf_scored.cpp:29-83).  Output lists are SoA:
// lists[(((b*C + c)*2 + dir)*7 + comp)*hw + pos], dir 0 = forward, 1 = backward.
__global__ void __launch_bounds__(NT) k_caf_scored(const float* __restrict__ caf, Dims d,
                                                   const int* __restrict__ skeleton,
                                                   const float* __restrict__ cifhr,
                                                   const unsigned* __restrict__ tile_epoch, unsigned epoch,
                                                   double revision,
                                                   double score_th, double cif_floor, int no_rescore,
                                                   float* __restrict__ lists, int* __restrict__ list_counts) {
    __shared__ int wc[NW];
    const int c = blockIdx.x, b = blockIdx.y;
    const float* cf = caf + ((size_t)(b * d.C + c) * 8) * d.hw;
    HrView hv;
    hv.hr = cifhr + (size_t)b * d.F * d.H * d.Wp;
    hv.tiles_x = d.tiles_x; hv.tiles = d.tiles_x * d.tiles_y;
    hv.tile_epoch = tile_epoch + (size_t)b * d.F * hv.tiles; hv.epoch = epoch;
    hv.F = d.F; hv.H = d.H; hv.W = d.W; hv.Wp = d.Wp;
    float* fw = lists + ((size_t)((b * d.C + c) * 2 + 0) * 7) * d.hw;
    float* bw = lists + ((size_t)((b * d.C + c) * 2 + 1) * 7) * d.hw;
    const long long kp_a = skeleton[2 * c], kp_b = skeleton[2 * c + 1];
    int nf = 0, nb = 0;
    for (int start = 0; start < d.hw; start += NT) {
        const int idx = start + threadIdx.x;
        bool ff = false, bf = false;
        float x1 = 0.f, y1 = 0.f, x2 = 0.f, y2 = 0.f, s1 = 0.f, s2 = 0.f, cfw = 0.f, cbw = 0.f;
        if (idx < d.hw) {
            const float cc = cf[1 * d.hw + idx];
            if (!((double)cc < score_th)) {
                const float st = (float)d.caf_stride;
                x1 = cf[2 * d.hw + idx] * st; y1 = cf[3 * d.hw + idx] * st;
                x2 = cf[4 * d.hw + idx] * st; y2 = cf[5 * d.hw + idx] * st;
                s1 = cf[6 * d.hw + idx] * st; s2 = cf[7 * d.hw + idx] * st;
                cfw = cc; cbw = cc;
                if (!no_rescore) {
                    const float fhr = cifhr_value(hv, revision, kp_b, x2, y2, 0.0f);
                    const float bhr = cifhr_value(hv, revision, kp_a, x1, y1, 0.0f);
                    cfw = (float)((double)cc * (cif_floor + (1.0 - cif_floor) * (double)fhr));
                    cbw = (float)((double)cc * (cif_floor + (1.0 - cif_floor) * (double)bhr));
                }
                ff = (double)cfw > score_th;
                bf = (double)cbw > score_th;
            }
        }
        int pf, pb;
        block_compact2<NW>(ff, bf, nf, nb, pf, pb, wc);
        if (ff) {
            fw[0 * d.hw + pf] = cfw; fw[1 * d.hw + pf] = x1; fw[2 * d.hw + pf] = y1;
            fw[3 * d.hw + pf] = x2; fw[4 * d.hw + pf] = y2; fw[5 * d.hw + pf] = s1; fw[6 * d.hw + pf] = s2;
        }
        if (bf) {
            bw[0 * d.hw + pb] = cbw; bw[1 * d.hw + pb] = x2; bw[2 * d.hw + pb] = y2;
            bw[3 * d.hw + pb] = x1; bw[4 * d.hw + pb] = y1; bw[5 * d.hw + pb] = s2; bw[6 * d.hw + pb] = s1;
        }
    }
    if (threadIdx.x == 0) {
        list_counts[(b * d.C + c) * 2 + 0] = nf;
        list_counts[(b * d.C + c) * 2 + 1] = nb;
    }
}

// ---------------------------------------------------------------------------
// grow_connection_blend (src/cifcaf.cpp:32-103), one warp per call.  The list is SoA: C0/X1/Y1 point at the scanned
// components (c, x_src, y_src), X2/Y2/S2 at the components read for the one or two winning entries (x_dst, y_dst,
// s_dst); both groups in shared memory when staged (a read of the winners from global memory is an L2 round trip on the
// serial path of every evaluation), n = the list's length.
// The reference's loop is order dependent (">=" shifts 1 -> 2, ">" replaces 2).  It is reproduced literally: the
// warp evaluates 32 entries at a time, then every lane replays the entries that passed the box filter -- in index
// order, values broadcast by shuffle -- through the same two-register update.  Few entries pass (the filter box is
// one joint scale wide), so the replay is short; no score cache, no reduction tree, any list length.
struct Joint { double v, x, y, s; };

__device__ Joint warp_blend(const float* C0, const float* X1, const float* Y1,
                            const float* X2, const float* Y2, const float* S2, int n,
                            double x, double y, double xy_scale, double filter_sigmas, bool only_max, int lane,
                            int* cand) {
    // cand: 32 ints of per-warp scratch (shared memory).  Two phases per round: (A) the cheap box test over the list, the
    // indices of the entries that pass compacted -- in index order -- into cand; (B) ONE pass of the expensive part
    // (double division, exp) with lane k on the k-th candidate, then the in-order replay.  A list whose 32-entry chunks
    // each hold a passing entry used to pay the double chain once per chunk (1-2 times per scan, two scans per
    // evaluation); the per-entry arithmetic and the replay order are unchanged.
    Joint zero; zero.v = 0.0; zero.x = 0.0; zero.y = 0.0; zero.s = 0.0;
    xy_scale = fmax(xy_scale, 0.5);
    const float sigma_filter = (float)(filter_sigmas * xy_scale / 2.0);
    const float sigma2 = (float)(0.25 * xy_scale * xy_scale);
    const double xlo = x - (double)sigma_filter, xhi = x + (double)sigma_filter;
    const double ylo = y - (double)sigma_filter, yhi = y + (double)sigma_filter;
    float score_1 = 0.0f, score_2 = 0.0f;
    int i1 = 0, i2 = 0;
    const unsigned lt = (1u << lane) - 1u;
    int base = 0;
    while (base < n) {
        int cnt = 0, next = base;
        for (; next < n; next += 32) {
            const int i = next + lane;
            bool pass = false;
            if (i < n) {
                const float ex = X1[i], ey = Y1[i];
                pass = !((double)ex < xlo) && !((double)ex > xhi) && !((double)ey < ylo) && !((double)ey > yhi);
            }
            const unsigned mask = __ballot_sync(0xffffffffu, pass);
            const int pc = __popc(mask);
            if (cnt + pc > 32) break;                 // does not fit any more: this chunk is scanned again next round
            if (pass) cand[cnt + __popc(mask & lt)] = i;
            cnt += pc;
        }
        __syncwarp();
        float sc = 0.0f;
        int ci = 0;
        if (lane < cnt) {
            ci = cand[lane];
            const double dx = (double)X1[ci] - x, dy = (double)Y1[ci] - y;
            const float d2 = (float)(dx * dx + dy * dy);
            sc = (float)(exp(-0.5 * (double)d2 / (double)sigma2) * (double)C0[ci]);
        }
        __syncwarp();
        for (int l = 0; l < cnt; l++) {
            const float v = __shfl_sync(0xffffffffu, sc, l);
            const int vi = __shfl_sync(0xffffffffu, ci, l);
            if (v >= score_1) { score_2 = score_1; i2 = i1; score_1 = v; i1 = vi; }
            else if (v > score_2) { score_2 = v; i2 = vi; }
        }
        base = next;
    }
    if (score_1 == 0.0f) return zero;
    const float e1x = X2[i1], e1y = Y2[i1];
    const float e1s = fmaxf(0.0f, S2[i1]);
    Joint r;
    if (only_max) { r.v = score_1; r.x = e1x; r.y = e1y; r.s = e1s; return r; }
    if ((double)score_2 < 0.01 || (double)score_2 < 0.5 * (double)score_1) {
        r.v = 0.5 * (double)score_1; r.x = e1x; r.y = e1y; r.s = e1s; return r;
    }
    const float e2x = X2[i2], e2y = Y2[i2];
    const float e2s = fmaxf(0.0f, S2[i2]);
    const double bdx = (double)(e1x - e2x), bdy = (double)(e1y - e2y);
    const float blend_d2 = (float)(bdx * bdx + bdy * bdy);
    if ((double)blend_d2 > ((double)e1s * (double)e1s) / 4.0) {
        r.v = 0.5 * (double)score_1; r.x = e1x; r.y = e1y; r.s = e1s; return r;
    }
    r.v = 0.5 * (double)(score_1 + score_2);
    r.x = (score_1 * e1x + score_2 * e2x) / (score_1 + score_2);
    r.y = (score_1 * e1y + score_2 * e2y) / (score_1 + score_2);
    r.s = (score_1 * e1s + score_2 * e2s) / (score_1 + score_2);
    return r;
}

// A joint as the workers keep it: x, y, s of the reference's double Joint (cifcaf.hpp:21-28) only ever hold float
// values (they come from float fields, float initial annotations or the float blend above), v is a true double.
struct WJoint { double v; float x, y, s; int pad; };
static_assert(sizeof(WJoint) == 24, "WJoint layout");

// Image-wide read-only context of a grow CTA (graph tables and CAF lists staged in shared memory).
struct GrowShared {
    const int* skeleton;    // [2C]
    const int* adj_start;   // [K+1]
    const int* adj_edge;    // [<=2C] directed edge ids (2*c + dir, start = skeleton[c][dir]) in skeleton order
    const int* edge_lookup; // [2C]: caf_i*2 + forward  (first-match rule of src/cifcaf.cpp:360-373)
    const int* pair_id;     // [2C]: canonical id of the (start,end) pair for in_frontier
    const float* s_cxy;     // [3][list_cap] staged (c, x_src, y_src)
    const float* s_ext;     // [3][ext_cap] staged (x_dst, y_dst, s_dst) of the lists that end below ext_cap
    const int* s_loff;      // [2C] offset in s_cxy or -1
    int list_cap, ext_cap;
    const float* lists;     // image base: [C][2][7][hw]
    const int* list_counts; // image base: [C][2]
    int K, C, F, hw;
    GrowParams gp;
};

// One warp's private working set: the annotation being grown and its frontier (src/cifcaf.hpp:91-94).
struct Worker {
    WJoint* joints;         // [K]
    WJoint* eval;           // [2C] eagerly evaluated _connection_value per directed edge
    float* heap_score;      // [2C + 1]
    int* heap_item;         // [2C + 1]: edge | computed << 30
    int* new_edges;         // [2C]
    unsigned char* in_frontier;   // [2C] by pair id
    int* cand;              // [32] scratch of warp_blend
    int heap_n, n_new;      // lane 0's registers
};

__host__ __device__ inline size_t worker_bytes(int K, int C) {
    size_t b = sizeof(WJoint) * (size_t)K + sizeof(WJoint) * 2 * (size_t)C + (sizeof(float) + 2 * sizeof(int)) * (2 * (size_t)C + 2)
               + ((2 * (size_t)C + 3) & ~(size_t)3) + 32 * sizeof(int);
    return (b + 15) & ~(size_t)15;
}

__device__ inline void worker_init(Worker& w, unsigned char* base, int K, int C) {
    size_t off = 0;
    w.joints = reinterpret_cast<WJoint*>(base + off); off += sizeof(WJoint) * K;
    w.eval = reinterpret_cast<WJoint*>(base + off); off += sizeof(WJoint) * 2 * C;
    w.heap_score = reinterpret_cast<float*>(base + off); off += sizeof(float) * (2 * C + 2);
    w.heap_item = reinterpret_cast<int*>(base + off); off += sizeof(int) * (2 * C + 2);
    w.new_edges = reinterpret_cast<int*>(base + off); off += sizeof(int) * (2 * C + 2);
    w.in_frontier = base + off; off += (2 * (size_t)C + 3) & ~(size_t)3;
    w.cand = reinterpret_cast<int*>(base + off);
    w.heap_n = 0; w.n_new = 0;
}

__device__ __forceinline__ bool heap_less(float a, float b) { return a < b; }   // src/cifcaf.cpp:27-29

// libstdc++ std::push_heap / std::pop_heap restated (bits/stl_heap.h), single thread.
__device__ void heap_push(Worker& g, float score, int item) {
    int hole = g.heap_n++;
    int parent = (hole - 1) / 2;
    while (hole > 0 && heap_less(g.heap_score[parent], score)) {
        g.heap_score[hole] = g.heap_score[parent];
        g.heap_item[hole] = g.heap_item[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    g.heap_score[hole] = score;
    g.heap_item[hole] = item;
}

__device__ void heap_pop(Worker& g, float& top_score, int& top_item) {
    top_score = g.heap_score[0];
    top_item = g.heap_item[0];
    const int n = g.heap_n;
    if (n > 1) {
        const int len = n - 1;
        const float vs = g.heap_score[len];
        const int vi = g.heap_item[len];
        int hole = 0, second = 0;
        while (second < (len - 1) / 2) {
            second = 2 * (second + 1);
            if (heap_less(g.heap_score[second], g.heap_score[second - 1])) second--;
            g.heap_score[hole] = g.heap_score[second];
            g.heap_item[hole] = g.heap_item[second];
            hole = second;
        }
        if ((len & 1) == 0 && second == (len - 2) / 2) {
            second = 2 * (second + 1);
            g.heap_score[hole] = g.heap_score[second - 1];
            g.heap_item[hole] = g.heap_item[second - 1];
            hole = second - 1;
        }
        int parent = (hole - 1) / 2;
        while (hole > 0 && heap_less(g.heap_score[parent], vs)) {
            g.heap_score[hole] = g.heap_score[parent];
            g.heap_item[hole] = g.heap_item[parent];
            hole = parent;
            parent = (hole - 1) / 2;
        }
        g.heap_score[hole] = vs;
        g.heap_item[hole] = vi;
    }
    g.heap_n = n - 1;
}

// src/cifcaf.cpp:316-346 (single thread)
__device__ void frontier_add_from(const GrowShared& g, Worker& w, int start_i) {
    const float max_score = (float)sqrt(w.joints[start_i].v);
    for (int a = g.adj_start[start_i]; a < g.adj_start[start_i + 1]; a++) {
        const int edge = g.adj_edge[a];
        const int c = edge >> 1, dir = edge & 1;
        const int end_i = g.skeleton[2 * c + (1 - dir)];
        if (w.joints[end_i].v > 0.0) continue;
        const int pid = g.pair_id[edge];
        if (w.in_frontier[pid]) continue;
        heap_push(w, max_score, edge);
        w.in_frontier[pid] = 1;
        w.new_edges[w.n_new++] = edge;
    }
}

// src/cifcaf.cpp:349-411, one warp
__device__ WJoint warp_connection_value(const GrowShared& g, const Worker& w, int edge, bool reverse_match_,
                                        double filter_sigmas, int lane) {
    const int c = edge >> 1, dir = edge & 1;
    const int start_i = g.skeleton[2 * c + dir];
    const int lk = g.edge_lookup[edge];
    const int caf_i = lk >> 1;
    const int forward = lk & 1;
    const int lif = caf_i * 2 + (forward ? 0 : 1), lib = caf_i * 2 + (forward ? 1 : 0);
    const float* Lf = g.lists + ((size_t)lif * 7) * g.hw;
    const float* Lb = g.lists + ((size_t)lib * 7) * g.hw;
    const int nf = g.list_counts[lif], nb = g.list_counts[lib];
    const WJoint sj = w.joints[start_i];
    const int of = g.s_loff[lif], ob = g.s_loff[lib];
    const float* fC = of >= 0 ? g.s_cxy + of : Lf;
    const float* fX = of >= 0 ? g.s_cxy + g.list_cap + of : Lf + g.hw;
    const float* fY = of >= 0 ? g.s_cxy + 2 * g.list_cap + of : Lf + 2 * (size_t)g.hw;
    const bool fe = of >= 0 && of + nf <= g.ext_cap;
    const float* fX2 = fe ? g.s_ext + of : Lf + 3 * (size_t)g.hw;
    const float* fY2 = fe ? g.s_ext + g.ext_cap + of : Lf + 4 * (size_t)g.hw;
    const float* fS2 = fe ? g.s_ext + 2 * g.ext_cap + of : Lf + 6 * (size_t)g.hw;
    WJoint out; out.v = 0.0; out.x = 0.f; out.y = 0.f; out.s = 0.f; out.pad = 0;
    const Joint nj = warp_blend(fC, fX, fY, fX2, fY2, fS2, nf, (double)sj.x, (double)sj.y, (double)sj.s, filter_sigmas, false, lane,
                                w.cand);
    if (nj.v == 0.0) return out;
    double v = sqrt(nj.v * sj.v);
    if (v < g.gp.keypoint_threshold || v < sj.v * g.gp.keypoint_threshold_rel) return out;
    if (g.gp.reverse_match && reverse_match_ && start_i < g.F) {
        const float* bC = ob >= 0 ? g.s_cxy + ob : Lb;
        const float* bX = ob >= 0 ? g.s_cxy + g.list_cap + ob : Lb + g.hw;
        const float* bY = ob >= 0 ? g.s_cxy + 2 * g.list_cap + ob : Lb + 2 * (size_t)g.hw;
        const bool be = ob >= 0 && ob + nb <= g.ext_cap;
        const float* bX2 = be ? g.s_ext + ob : Lb + 3 * (size_t)g.hw;
        const float* bY2 = be ? g.s_ext + g.ext_cap + ob : Lb + 4 * (size_t)g.hw;
        const float* bS2 = be ? g.s_ext + 2 * g.ext_cap + ob : Lb + 6 * (size_t)g.hw;
        const Joint rev = warp_blend(bC, bX, bY, bX2, bY2, bS2, nb, nj.x, nj.y, nj.s, filter_sigmas, false, lane, w.cand);
        if (rev.v == 0.0) return out;
        if (fabs((double)sj.x - rev.x) + fabs((double)sj.y - rev.y) > (double)sj.s) return out;
    }
    out.v = v; out.x = (float)nj.x; out.y = (float)nj.y; out.s = (float)nj.s;
    return out;
}

// src/cifcaf.cpp:265-313 (_grow) and :429-449 (_flood_fill when flood == true).  One WARP grows one annotation
// (w.joints): lane 0 drives the libstdc++-order heap, the whole warp evaluates the CAF scans behind the frontier
// entries as they are added.  Warp-synchronous: no CTA barrier inside.
__device__ void warp_grow(const GrowShared& g, Worker& w, bool reverse_match_, double filter_sigmas, bool flood, int lane) {
    __syncwarp();
    for (int i = lane; i < 2 * g.C; i += 32) w.in_frontier[i] = 0;
    __syncwarp();
    w.heap_n = 0; w.n_new = 0;
    if (lane == 0) {
        for (int j = 0; j < g.K; j++) {
            if (w.joints[j].v == 0.0) continue;
            frontier_add_from(g, w, j);
        }
    }
    for (;;) {
        __syncwarp();
        const int n_new = __shfl_sync(0xffffffffu, w.n_new, 0);
        if (!flood) {
            for (int e = 0; e < n_new; e++) {
                const int edge = w.new_edges[e];
                const WJoint r = warp_connection_value(g, w, edge, reverse_match_, filter_sigmas, lane);
                if (lane == 0) w.eval[edge] = r;
            }
        }
        __syncwarp();
        int done = 0;
        if (lane == 0) {
            w.n_new = 0;
            while (w.heap_n > 0 && w.n_new == 0) {
                float score; int item;
                heap_pop(w, score, item);
                const int edge = item & 0x3fffffff;
                const bool computed = (item >> 30) & 1;
                const int c = edge >> 1, dir = edge & 1;
                const int start_i = g.skeleton[2 * c + dir];
                const int end_i = g.skeleton[2 * c + (1 - dir)];
                if (w.joints[end_i].v > 0.0) continue;
                if (flood) {
                    WJoint nj = w.joints[start_i];
                    nj.v = 0.00001;
                    w.joints[end_i] = nj;
                    frontier_add_from(g, w, end_i);
                    w.n_new = 0;           // nothing to evaluate in flood mode
                    continue;
                }
                const WJoint nj = w.eval[edge];
                if (!computed) {
                    if (nj.v == 0.0) continue;     // block_joints has no effect (src/cifcaf.cpp:291-295)
                    if (!g.gp.greedy) {
                        heap_push(w, (float)nj.v, edge | (1 << 30));
                        continue;
                    }
                }
                w.joints[end_i] = nj;
                frontier_add_from(g, w, end_i);
            }
            done = (w.heap_n == 0 && w.n_new == 0) ? 1 : 0;
        }
        done = __shfl_sync(0xffffffffu, done, 0);
        if (done) break;
    }
    __syncwarp();
}

// Occupancy (src/occupancy.cpp:13-43) on a byte map with epoch tags.
struct Occ {
    unsigned char* map;   // image base [F][Ho][Wo]
    int F, Ho, Wo;
    double reduction, min_scale_reduced;
    unsigned char tag;
};

__device__ __forceinline__ void occ_cell(const Occ& o, double x, double y, long long& xi, long long& yi) {
    if (o.reduction != 1.0) { x /= o.reduction; y /= o.reduction; }
    xi = clamp_ll((long long)x, 0, o.Wo - 1);
    yi = clamp_ll((long long)y, 0, o.Ho - 1);
}

__device__ __forceinline__ bool occ_get(const Occ& o, long long f, double x, double y) {
    if (f >= o.F) return true;
    long long xi, yi;
    occ_cell(o, x, y, xi, yi);
    return reinterpret_cast<const volatile unsigned char*>(o.map)[((size_t)f * o.Ho + yi) * o.Wo + xi] == o.tag;
}

__device__ __forceinline__ void occ_box(const Occ& o, double x, double y, double sigma,
                                        long long& minx, long long& miny, long long& maxx, long long& maxy) {
    if (o.reduction != 1.0) {
        x /= o.reduction; y /= o.reduction;
        sigma = fmax(o.min_scale_reduced, sigma / o.reduction);
    }
    minx = clamp_ll((long long)(x - sigma), 0, o.Wo - 1);
    miny = clamp_ll((long long)(y - sigma), 0, o.Ho - 1);
    maxx = clamp_ll((long long)(x + sigma), minx + 1, o.Wo);
    maxy = clamp_ll((long long)(y + sigma), miny + 1, o.Ho);
}

// one warp fills the box
__device__ __forceinline__ void occ_set_warp(const Occ& o, long long f, double x, double y, double sigma, int lane) {
    long long minx, miny, maxx, maxy;
    occ_box(o, x, y, sigma, minx, miny, maxx, maxy);
    const int bw = (int)(maxx - minx), bh = (int)(maxy - miny);
    volatile unsigned char* base = o.map + ((size_t)f * o.Ho + miny) * o.Wo + minx;
    for (int k = lane; k < bw * bh; k += 32) base[(size_t)(k / bw) * o.Wo + (k % bw)] = o.tag;
}

// would occupancy.get(f, x, y) see a cell that occupancy.set of joint j (field f) marks?  (exact box arithmetic)
__device__ __forceinline__ bool occ_joint_covers(const Occ& o, const WJoint& j, double x, double y) {
    if (j.v == 0.0) return false;
    long long xi, yi, minx, miny, maxx, maxy;
    occ_cell(o, x, y, xi, yi);
    occ_box(o, (double)j.x, (double)j.y, (double)j.s, minx, miny, maxx, maxy);
    return xi >= minx && xi < maxx && yi >= miny && yi < maxy;
}

constexpr int GROW_MAX_WORKERS = 16;       // warps per grow CTA == annotations grown concurrently per image

struct GrowLayout { int workers, list_cap, ext_cap; size_t smem; };

// shared memory plan of a grow CTA: graph tables | list offsets | staged lists | per-warp workers | control
__host__ __device__ inline size_t grow_fixed_bytes(int K, int C) {
    return (((size_t)(8 * C + K + 1 + 2 * C + 2 * C + 8) * sizeof(int)) + 15) & ~(size_t)15;
}

inline GrowLayout plan_grow(int K, int C) {
    const size_t budget = 200 * 1024, fixed = grow_fixed_bytes(K, C) + 64 * sizeof(int) + 256;
    const size_t wb = worker_bytes(K, C);
    GrowLayout l;
    l.list_cap = LIST_SMEM_ENTRIES;
    size_t lists = sizeof(float) * 3 * (size_t)l.list_cap;
    if (fixed + lists + 4 * wb > budget) { l.list_cap = LIST_SMEM_ENTRIES / 2; lists /= 2; }
    long w = (long)((budget - fixed - lists) / wb);
    l.workers = (int)std::max(1L, std::min((long)GROW_MAX_WORKERS, w));
    // what is left stages the destination components (x_dst, y_dst, s_dst) of the first ext_cap entries
    const size_t used = fixed + lists + (size_t)l.workers * wb;
    long ext = used < budget ? (long)((budget - used) / (3 * sizeof(float))) : 0;
    l.ext_cap = (int)std::max(0L, std::min((long)l.list_cap, ext / 32 * 32));
    l.smem = used + sizeof(float) * 3 * (size_t)l.ext_cap;
    return l;
}

struct Graph {
    const int* skeleton; const int* adj_start; const int* adj_edge; const int* edge_lookup; const int* pair_id;
};

// carve the CTA's shared memory, stage the graph tables and the scanned list components; whole CTA
__device__ void grow_shared_init(GrowShared& g, unsigned char* smem, const Graph& gr, const Dims& d, int list_cap, int ext_cap,
                                 const float* lists, const int* list_counts, const GrowParams& gp,
                                 unsigned char** workers_base, int** ctl) {
    const int K = d.K, C = d.C;
    int* tab = reinterpret_cast<int*>(smem);
    int* s_skel = tab;                    // 2C
    int* s_adj_start = s_skel + 2 * C;    // K + 1
    int* s_adj_edge = s_adj_start + K + 1;   // 2C
    int* s_lookup = s_adj_edge + 2 * C;   // 2C
    int* s_pair = s_lookup + 2 * C;       // 2C
    int* s_loff = s_pair + 2 * C;         // 2C
    int* s_lcnt = s_loff + 2 * C;         // 2C: list lengths (read on the serial path of every evaluation)
    int* s_ctl = s_lcnt + 2 * C;          // 8
    unsigned char* p = smem + grow_fixed_bytes(K, C);
    float* s_cxy = reinterpret_cast<float*>(p);
    p += sizeof(float) * 3 * (size_t)list_cap;
    float* s_ext = reinterpret_cast<float*>(p);
    p += sizeof(float) * 3 * (size_t)ext_cap;
    *workers_base = p;
    *ctl = s_ctl;
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
        s_skel[i] = gr.skeleton[i]; s_lookup[i] = gr.edge_lookup[i]; s_pair[i] = gr.pair_id[i];
    }
    for (int i = threadIdx.x; i <= K; i += blockDim.x) s_adj_start[i] = gr.adj_start[i];
    __syncthreads();
    for (int i = threadIdx.x; i < s_adj_start[K]; i += blockDim.x) s_adj_edge[i] = gr.adj_edge[i];
    // list offsets in the staging area: counts fetched in parallel (s_loff doubles as scratch), then one thread runs
    // the greedy first-fit prefix over shared memory (a serial walk over global memory pays one
    // load latency per list: 38 lists for COCO, 320 for the wholebody skeleton)
    for (int li = threadIdx.x; li < 2 * C; li += blockDim.x) { const int n = list_counts[li]; s_loff[li] = n; s_lcnt[li] = n; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int li = 0; li < 2 * C; li++) {
            const int n = s_loff[li];
            if (run + n <= list_cap) { s_loff[li] = run; run += n; }
            else s_loff[li] = -1;
        }
    }
    __syncthreads();
    // one warp per list (lists are short: a few dozen entries)
    {
        const int warp_i = threadIdx.x >> 5, lane_i = threadIdx.x & 31, n_warps = blockDim.x >> 5;
        for (int li = warp_i; li < 2 * C; li += n_warps) {
            const int off = s_loff[li];
            if (off < 0) continue;
            const int n = s_lcnt[li];
            const float* L = lists + ((size_t)li * 7) * d.hw;
            for (int i = lane_i; i < n; i += 32) {
                s_cxy[off + i] = L[i];
                s_cxy[list_cap + off + i] = L[d.hw + i];
                s_cxy[2 * list_cap + off + i] = L[2 * (size_t)d.hw + i];
            }
            if (off + n <= ext_cap) {
                for (int i = lane_i; i < n; i += 32) {
                    s_ext[off + i] = L[3 * (size_t)d.hw + i];
                    s_ext[ext_cap + off + i] = L[4 * (size_t)d.hw + i];
                    s_ext[2 * ext_cap + off + i] = L[6 * (size_t)d.hw + i];
                }
            }
        }
    }
    g.skeleton = s_skel; g.adj_start = s_adj_start; g.adj_edge = s_adj_edge; g.edge_lookup = s_lookup; g.pair_id = s_pair;
    g.s_cxy = s_cxy; g.s_ext = s_ext; g.s_loff = s_loff; g.list_cap = list_cap; g.ext_cap = ext_cap;
    g.lists = lists; g.list_counts = s_lcnt;
    g.K = K; g.C = C; g.F = d.F; g.hw = d.hw; g.gp = gp;
    __syncthreads();
}

// Seed loop of CifCaf::call_with_initial_annotations (src/cifcaf.cpp:173-231).  One CTA per image, one WARP per
// annotation in flight.  The reference is sequential only through the occupancy map: a seed is skipped if an earlier
// annotation covers it, and _grow itself reads nothing but the seed and the (static) CAF lists.  So every round
//   1. selects the next W seeds, in order, that the occupancy map does not cover yet,
//   2. grows all W speculatively, one per warp,
//   3. commits them in seed order: seed i is dropped iff a joint of an annotation committed earlier IN THIS ROUND
//      covers it (the same box arithmetic as Occupancy::set/get), else it marks the map and is stored,
// which yields exactly the annotations, in exactly the order, of the sequential loop.
__global__ void __launch_bounds__(32 * GROW_MAX_WORKERS) k_grow(Dims d, Graph gr, GrowParams gp, int list_cap, int ext_cap,
                                             const int* __restrict__ seed_f, const float4* __restrict__ seed_vxys,
                                             const int* __restrict__ n_seeds,
                                             const float* __restrict__ lists, const int* __restrict__ list_counts,
                                             unsigned char* __restrict__ occ_map, unsigned char occ_tag,
                                             const float* __restrict__ init_ann, const long long* __restrict__ init_ids,
                                             const int* __restrict__ init_counts, int init_cap,
                                             Joint* __restrict__ anns, long long* __restrict__ ann_ids,
                                             int* __restrict__ n_anns, int* __restrict__ flags,
                                             long long* __restrict__ dbg) {
    // dbg (diagnostics, may be null): per image 6 values -- rounds, picks, clocks in init / select / grow / commit
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_sel[GROW_MAX_WORKERS];       // seed index (or initial-annotation index) per worker
    __shared__ int s_slot[GROW_MAX_WORKERS];      // output slot, or -1 if dropped
    __shared__ int s_wc[GROW_MAX_WORKERS];
    __shared__ float s_px[GROW_MAX_WORKERS], s_py[GROW_MAX_WORKERS], s_pr[GROW_MAX_WORKERS];   // picks: x, y, scale
    __shared__ unsigned char s_cov[GROW_MAX_WORKERS][GROW_MAX_WORKERS];   // annotation a covers the seed of pick i
    __shared__ int s_nsel, s_ptr, s_nann, s_over, s_scan_end, s_stop;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int W = blockDim.x >> 5;
    GrowShared g;
    unsigned char* workers_base; int* ctl;
    long long t_mark = clock64(), t_init = 0, t_sel = 0, t_grow = 0, t_commit = 0;
    int n_rounds = 0, n_picks = 0;
    auto lap = [&](long long& acc) { const long long now = clock64(); acc += now - t_mark; t_mark = now; };
    grow_shared_init(g, smem, gr, d, list_cap, ext_cap, lists + ((size_t)b * d.C * 2 * 7) * d.hw,
                     list_counts + (size_t)b * d.C * 2, gp, &workers_base, &ctl);
    (void)ctl;
    Worker w;
    worker_init(w, workers_base + (size_t)warp * worker_bytes(d.K, d.C), d.K, d.C);
    lap(t_init);
    // every warp can read every worker's joints at commit time
    auto joints_of = [&](int wk) { return reinterpret_cast<const WJoint*>(workers_base + (size_t)wk * worker_bytes(d.K, d.C)); };

    Occ occ;
    occ.map = occ_map + (size_t)b * d.F * d.Ho * d.Wo;
    occ.F = d.F; occ.Ho = d.Ho; occ.Wo = d.Wo;
    occ.reduction = gp.occ_reduction; occ.min_scale_reduced = gp.occ_min_scale_reduced;
    occ.tag = occ_tag;

    Joint* my_anns = anns + (size_t)b * d.max_ann * d.K;
    long long* my_ids = ann_ids + (size_t)b * d.max_ann;
    const int ns = n_seeds[b];
    const int* sf = seed_f + (size_t)b * d.F * d.hw;
    const float4* sv = seed_vxys + (size_t)b * d.F * d.hw;
    const int n_init = (init_ann != nullptr && init_counts != nullptr) ? init_counts[b] : 0;
    if (tid == 0) { s_ptr = 0; s_nann = 0; s_over = 0; }
    __syncthreads();

    // store + occupancy marks of the annotation this warp grew (src/cifcaf.cpp:196-201, 225-230)
    auto commit_mine = [&](int slot, long long id) {
        for (int of = 0; of < d.F && of < d.K; of++) {
            const WJoint j = w.joints[of];
            if (j.v == 0.0) continue;
            occ_set_warp(occ, of, (double)j.x, (double)j.y, (double)j.s, lane);
        }
        for (int k = lane; k < d.K; k += 32) {
            const WJoint j = w.joints[k];
            Joint o; o.v = j.v; o.x = (double)j.x; o.y = (double)j.y; o.s = (double)j.s;
            my_anns[(size_t)slot * d.K + k] = o;
        }
        if (lane == 0) my_ids[slot] = id;
    };

    // ---- initial annotations (src/cifcaf.cpp:177-202): always kept, W at a time
    for (int a0 = 0; a0 < n_init && !s_over; a0 += W) {
        const int a = a0 + warp;
        const bool mine = a < n_init && s_nann + warp < d.max_ann;
        if (mine) {
            for (int k = lane; k < d.K; k += 32) {
                const float* s = init_ann + (((size_t)b * init_cap + a) * d.K + k) * 4;
                WJoint j; j.v = (double)s[0]; j.x = s[1]; j.y = s[2]; j.s = s[3]; j.pad = 0;
                w.joints[k] = j;
            }
            warp_grow(g, w, true, 1.0, false, lane);
            commit_mine(s_nann + warp, init_ids[(size_t)b * init_cap + a]);
        }
        __syncthreads();
        if (tid == 0) {
            const int n = min(W, n_init - a0);
            if (s_nann + n > d.max_ann) { s_over = 1; s_nann = d.max_ann; } else s_nann += n;
        }
        __syncthreads();
    }

    // ---- seeds
    // Round structure with DEFERRAL.  The seeds of one person crowd the top of the sorted list (every joint casts
    // a dozen high seeds), so "the next W uncovered seeds" would mostly be W seeds of the same one or two people,
    // all but the first dropped at commit time.  A seed close to a seed already picked in this round is therefore
    // DEFERRED: not grown now, in the expectation that the picked neighbour's annotation will cover it.  The commit
    // walk stays exact: seeds are resolved strictly in order; the first deferred seed that turns out NOT to be
    // covered by the annotations committed before it stops the walk (s_ptr = that seed; later picks of this round
    // are thrown away and re-examined in the next round, which picks that seed first).  The heuristic only decides
    // how much speculative work is wasted, never the result.
    const float defer_k = gp.defer_radius;
    while (!s_over) {
        // 1. selection: scan from s_ptr in chunks of blockDim seeds, in order
        if (tid == 0) { s_nsel = 0; s_scan_end = s_ptr; }
        __syncthreads();
        int ptr = s_ptr;
        while (ptr < ns) {
            const int idx = ptr + tid;
            bool avail = false;
            float4 sd = make_float4(0.f, 0.f, 0.f, 0.f);
            if (idx < ns) {
                sd = sv[idx];
                avail = !occ_get(occ, sf[idx], (double)sd.y, (double)sd.z);
            }
            int n_known = s_nsel;                 // picks of earlier chunks of this round
            if (avail && defer_k > 0.f)
                for (int k = 0; k < n_known && avail; k++) {
                    const float r = defer_k * fmaxf(s_pr[k], sd.w);
                    if (fabsf(sd.y - s_px[k]) <= r && fabsf(sd.z - s_py[k]) <= r) avail = false;
                }
            for (;;) {
                // first still-available seed of the chunk
                const unsigned m = __ballot_sync(0xffffffffu, avail);
                if (lane == 0) s_wc[warp] = m ? (warp * 32 + __ffs(m) - 1) : INT_MAX;
                __syncthreads();
                int first = INT_MAX;
                for (int w2 = 0; w2 < W; w2++) first = min(first, s_wc[w2]);
                if (first == INT_MAX) { __syncthreads(); break; }
                if (tid == first) {
                    const int k = s_nsel;
                    s_sel[k] = idx; s_px[k] = sd.y; s_py[k] = sd.z; s_pr[k] = sd.w;
                    s_nsel = k + 1;
                    avail = false;
                }
                __syncthreads();
                const int k = s_nsel - 1;
                if (avail && defer_k > 0.f) {
                    const float r = defer_k * fmaxf(s_pr[k], sd.w);
                    if (fabsf(sd.y - s_px[k]) <= r && fabsf(sd.z - s_py[k]) <= r) avail = false;
                }
                if (k + 1 == W) break;            // uniform
            }
            __syncthreads();
            if (s_nsel == W) { if (tid == 0) s_scan_end = s_sel[W - 1] + 1; break; }
            ptr += blockDim.x;
            if (tid == 0) s_scan_end = min(ptr, ns);
        }
        __syncthreads();
        const int n_sel = s_nsel;
        const int scan_end = s_scan_end;
        lap(t_sel);
        if (n_sel == 0) break;                    // every remaining seed is covered by the map
        n_rounds++; n_picks += n_sel;
        // 2. grow, one warp per picked seed
        if (warp < n_sel) {
            const int si = s_sel[warp];
            const float4 sd = sv[si];
            const int f = sf[si];
            for (int k = lane; k < d.K; k += 32) {
                WJoint j; j.v = 0.0; j.x = 0.f; j.y = 0.f; j.s = 0.f; j.pad = 0;
                if (k == f) { j.v = (double)sd.x; j.x = sd.y; j.y = sd.z; j.s = sd.w; }
                w.joints[k] = j;
            }
            warp_grow(g, w, true, 1.0, false, lane);
        }
        if (tid == 0) s_stop = INT_MAX;
        __syncthreads();
        lap(t_grow);
        // 3a. keep / drop of the picks among themselves, in seed order (picks are in ascending seed order): the
        // "annotation a would cover seed i" matrix in parallel, then the order-dependent walk over it
        if (tid < GROW_MAX_WORKERS * GROW_MAX_WORKERS) {
            const int i = tid / GROW_MAX_WORKERS, a = tid % GROW_MAX_WORKERS;
            bool c = false;
            if (a < i && i < n_sel) {
                const int si = s_sel[i];
                const float4 sd = sv[si];
                const int f = sf[si];
                if (f < d.F && f < d.K) c = occ_joint_covers(occ, joints_of(a)[f], (double)sd.y, (double)sd.z);
            }
            s_cov[i][a] = c ? 1 : 0;
        }
        __syncthreads();
        if (tid == 0) {
            for (int i = 0; i < n_sel; i++) {
                bool covered = false;
                for (int a = 0; a < i && !covered; a++) covered = s_slot[a] >= 0 && s_cov[i][a];
                s_slot[i] = covered ? -1 : 0;
            }
        }
        __syncthreads();
        // 3b. the first deferred seed that no earlier kept pick covers stops the walk
        for (int idx = s_ptr + tid; idx < scan_end; idx += blockDim.x) {
            bool is_pick = false;
            for (int k = 0; k < n_sel; k++) is_pick |= (s_sel[k] == idx);
            if (is_pick) continue;
            const float4 sd = sv[idx];
            const int f = sf[idx];
            if (occ_get(occ, f, (double)sd.y, (double)sd.z)) continue;        // covered by the map: resolved
            bool covered = false;
            if (f < d.F && f < d.K)
                for (int a = 0; a < n_sel && s_sel[a] < idx && !covered; a++) {
                    if (s_slot[a] < 0) continue;
                    covered = occ_joint_covers(occ, joints_of(a)[f], (double)sd.y, (double)sd.z);
                }
            if (!covered) atomicMin(&s_stop, idx);
        }
        __syncthreads();
        // 3c. output slots of the kept picks before the stop
        if (tid == 0) {
            const int stop = s_stop;
            int n_keep = 0;
            for (int i = 0; i < n_sel; i++) {
                if (s_slot[i] < 0) continue;
                if (s_sel[i] > stop) { s_slot[i] = -1; continue; }
                if (s_nann + n_keep >= d.max_ann) { s_over = 1; s_slot[i] = -1; continue; }
                s_slot[i] = s_nann + n_keep;
                n_keep++;
            }
            s_nann += n_keep;
            s_ptr = min(stop, scan_end);
        }
        __syncthreads();
        if (warp < n_sel && s_slot[warp] >= 0) commit_mine(s_slot[warp], -1);
        __syncthreads();          // occupancy marks visible to the next selection
        lap(t_commit);
        if (s_ptr >= ns) break;
    }
    if (dbg != nullptr && tid == 0) {
        long long* o = dbg + (size_t)b * 6;
        o[0] = n_rounds; o[1] = n_picks; o[2] = t_init; o[3] = t_sel; o[4] = t_grow; o[5] = t_commit;
    }
    if (tid == 0) {
        n_anns[b] = s_nann;
        flags[b] = s_over ? 1 : 0;
    }
}

// _force_complete + _flood_fill (src/cifcaf.cpp:233-236, 414-449); lists were refilled at force_complete_caf_th by
// k_caf_scored.  Annotations are independent here: one warp each, W at a time.
__global__ void __launch_bounds__(32 * GROW_MAX_WORKERS) k_force_complete(Dims d, Graph gr, GrowParams gp, int list_cap, int ext_cap,
                                                       const float* __restrict__ lists,
                                                       const int* __restrict__ list_counts,
                                                       Joint* __restrict__ anns, const int* __restrict__ n_anns) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int W = blockDim.x >> 5;
    GrowShared g;
    unsigned char* workers_base; int* ctl;
    grow_shared_init(g, smem, gr, d, list_cap, ext_cap, lists + ((size_t)b * d.C * 2 * 7) * d.hw,
                     list_counts + (size_t)b * d.C * 2, gp, &workers_base, &ctl);
    (void)ctl;
    Worker w;
    worker_init(w, workers_base + (size_t)warp * worker_bytes(d.K, d.C), d.K, d.C);
    Joint* my_anns = anns + (size_t)b * d.max_ann * d.K;
    const int n = n_anns[b];
    for (int a = warp; a < n; a += W) {
        for (int k = lane; k < d.K; k += 32) {
            const Joint j = my_anns[(size_t)a * d.K + k];
            WJoint o; o.v = j.v; o.x = (float)j.x; o.y = (float)j.y; o.s = (float)j.s; o.pad = 0;
            w.joints[k] = o;
        }
        warp_grow(g, w, false, 4.0, false, lane);
        warp_grow(g, w, false, 4.0, true, lane);
        for (int k = lane; k < d.K; k += 32) {
            const WJoint j = w.joints[k];
            Joint o; o.v = j.v; o.x = (double)j.x; o.y = (double)j.y; o.s = (double)j.s;
            my_anns[(size_t)a * d.K + k] = o;
        }
    }
}

// include/openpifpaf/decoder/utils/nms_keypoints.hpp:25-32
__device__ double uniform_score(const Joint* joints, int K) {
    double init = 0.0;
    for (int k = 0; k < K; k++) { const float i = (float)init; init = (double)i + joints[k].v; }
    return init / (double)K;
}

// NMSKeypoints::call (src/nms_keypoints.cpp:17-69) + output packing (src/cifcaf.cpp:246-261).
__global__ void __launch_bounds__(NT) k_nms(Dims d, GrowParams gp, Joint* __restrict__ anns,
                                            const long long* __restrict__ ann_ids, const int* __restrict__ n_anns,
                                            unsigned char* __restrict__ occ_map, unsigned char occ_tag,
                                            float4* __restrict__ out_ann, long long* __restrict__ out_ids,
                                            int* __restrict__ out_counts) {
    extern __shared__ __align__(16) unsigned char smem[];
    double* score = reinterpret_cast<double*>(smem);                 // [max_ann]
    int* order = reinterpret_cast<int*>(score + d.max_ann);          // [max_ann] sorted position -> annotation
    int* keep_rank = order + d.max_ann;                              // [max_ann]
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    Joint* my_anns = anns + (size_t)b * d.max_ann * d.K;
    const int n = n_anns[b];

    Occ occ;
    occ.map = occ_map + (size_t)b * d.F * d.Ho * d.Wo;
    occ.F = d.F; occ.Ho = d.Ho; occ.Wo = d.Wo;
    occ.reduction = gp.occ_reduction; occ.min_scale_reduced = gp.occ_min_scale_reduced;
    occ.tag = occ_tag;     // fresh tag == occupancy->clear() (src/nms_keypoints.cpp:18)

    for (int a = tid; a < n; a += NT) score[a] = uniform_score(my_anns + (size_t)a * d.K, d.K);
    __syncthreads();
    // std::sort descending; exact ties keep creation order
    for (int a = tid; a < n; a += NT) {
        const double s = score[a];
        int r = 0;
        for (int o = 0; o < n; o++) {
            const double so = score[o];
            if (so > s || (so == s && o < a)) r++;
        }
        order[r] = a;
    }
    __syncthreads();
    // occupancy planes of different keypoints are independent: one warp per field,
    // annotations in sorted order inside (src/nms_keypoints.cpp:29-45)
    for (int f = warp; f < d.K && f < d.F; f += NW) {
        for (int r = 0; r < n; r++) {
            Joint* jp = my_anns + (size_t)order[r] * d.K + f;
            const Joint j = *jp;
            if (j.v == 0.0) continue;
            if (occ_get(occ, f, j.x, j.y)) {
                if (lane == 0) jp->v = j.v * gp.nms_suppression;
            } else {
                occ_set_warp(occ, f, j.x, j.y, j.s, lane);
            }
            __syncwarp();
        }
    }
    __syncthreads();
    for (int i = tid; i < n * d.K; i += NT) {
        if (!(my_anns[i].v > gp.nms_keypoint_threshold)) my_anns[i].v = 0.0;
    }
    __syncthreads();
    for (int a = tid; a < n; a += NT) score[a] = uniform_score(my_anns + (size_t)a * d.K, d.K);
    __syncthreads();
    // remove_if(score < instance_threshold) keeps the first sort's order; second sort
    for (int r = tid; r < n; r += NT) {
        const int a = order[r];
        const double s = score[a];
        int kr = -1;
        if (!(s < gp.nms_instance_threshold)) {
            kr = 0;
            for (int r2 = 0; r2 < n; r2++) {
                const double so = score[order[r2]];
                if (so < gp.nms_instance_threshold) continue;
                if (so > s || (so == s && r2 < r)) kr++;
            }
        }
        keep_rank[a] = kr;
    }
    __syncthreads();
    int kept = 0;
    for (int a = 0; a < n; a++) kept += (keep_rank[a] >= 0) ? 1 : 0;     // uniform, n is small
    float4* my_out = out_ann + (size_t)b * d.max_ann * d.K;
    for (int i = tid; i < n * d.K; i += NT) {
        const int a = i / d.K, k = i % d.K;
        const int kr = keep_rank[a];
        if (kr < 0) continue;
        const Joint j = my_anns[(size_t)a * d.K + k];
        my_out[(size_t)kr * d.K + k] = make_float4((float)j.v, (float)j.x, (float)j.y, (float)j.s);
    }
    for (int a = tid; a < n; a += NT) {
        const int kr = keep_rank[a];
        if (kr >= 0) out_ids[(size_t)b * d.max_ann + kr] = ann_ids[(size_t)b * d.max_ann + a];
    }
    if (tid == 0) out_counts[b] = kept;
}

// Pack the results of all images into ONE device buffer so that a single small D2H copy fetches them:
//   int32 header: counts[B] | flags[B] | offsets[B+1]   (padded to 16 bytes)
//   records     : total x (K+1) float4 -- K joints (v,x,y,s) then {id (int64 bits in .x,.y), 0, 0}
__device__ __host__ inline size_t result_header_bytes(int B) { return ((size_t)(3 * B + 1) * 4 + 15) & ~(size_t)15; }

__global__ void __launch_bounds__(NT) k_pack(Dims d, const float4* __restrict__ out_ann,
                                             const long long* __restrict__ out_ids,
                                             const int* __restrict__ out_counts, const int* __restrict__ flags,
                                             unsigned char* __restrict__ result) {
    __shared__ int s_off;
    const int b = blockIdx.x, tid = threadIdx.x;
    int* hdr = reinterpret_cast<int*>(result);
    if (tid == 0) {
        int off = 0;
        for (int i = 0; i < b; i++) off += out_counts[i];
        s_off = off;
        hdr[b] = out_counts[b];
        hdr[d.B + b] = flags[b];
        hdr[2 * d.B + b] = off;
        if (b == d.B - 1) hdr[3 * d.B] = off + out_counts[b];
    }
    __syncthreads();
    const int off = s_off, n = out_counts[b];
    float4* rec = reinterpret_cast<float4*>(result + result_header_bytes(d.B));
    const float4* src = out_ann + (size_t)b * d.max_ann * d.K;
    const int R = d.K + 1;
    for (int i = tid; i < n * R; i += NT) {
        const int a = i / R, k = i - a * R;
        float4 v;
        if (k < d.K) {
            v = src[(size_t)a * d.K + k];
        } else {
            const long long id = out_ids[(size_t)b * d.max_ann + a];
            v = make_float4(__int_as_float((int)(id & 0xffffffffLL)), __int_as_float((int)(id >> 32)), 0.f, 0.f);
        }
        rec[(size_t)(off + a) * R + k] = v;
    }
}

__global__ void k_blend_single(const float* __restrict__ L, int n, double x, double y, double s,
                               double filter_sigmas, int only_max, double* __restrict__ out) {
    __shared__ int cand[32];
    const Joint j = warp_blend(L, L + n, L + 2 * (size_t)n, L + 3 * (size_t)n, L + 4 * (size_t)n, L + 6 * (size_t)n, n,
                               x, y, s, filter_sigmas, only_max != 0, threadIdx.x & 31, cand);
    if (threadIdx.x == 0) { out[0] = j.x; out[1] = j.y; out[2] = j.s; out[3] = j.v; }
}

// The dynamic shared-memory limit of a kernel is state of the kernel in the device's context, shared by every handle
// of the process.  Each handle only ever raises it: a handle created later with a smaller plan (another skeleton, a
// smaller detection capacity) must not lower it below what an older handle launches with.
cudaError_t raise_smem_limit(const void* kernel, int device, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, size_t> limit;
    std::lock_guard<std::mutex> lock(mu);
    size_t& cur = limit[{kernel, device}];
    if (bytes <= cur) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) cur = bytes;
    return e;
}

template <typename T>
int dev_alloc(T** p, size_t n) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), sizeof(T) * (n ? n : 1));
    if (e != cudaSuccess) {
        pifpaf::set_error("cudaMalloc of %zu bytes failed: %s", sizeof(T) * n, cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? PIFPAF_E_NOMEM : PIFPAF_E_CUDA;
    }
    return PIFPAF_OK;
}

}  // namespace

struct pifpaf_decoder {
    int device = 0;
    int K = 0, F = 0, C = 0;
    int max_batch = 0, max_h = 0, max_w = 0, max_stride = 0, max_ann = 0;
    std::vector<int64_t> skeleton;
    // graph
    int *d_skeleton = nullptr, *d_adj_start = nullptr, *d_adj_edge = nullptr, *d_edge_lookup = nullptr, *d_pair_id = nullptr;
    // workspace
    float* d_cifhr = nullptr;
    float4* d_cells = nullptr; int4* d_boxes = nullptr; int* d_cell_counts = nullptr;
    unsigned* d_tile_epoch = nullptr; int* d_worklist = nullptr; int* d_work_count = nullptr;
    unsigned hr_epoch = 0; size_t tile_epoch_elems = 0; int n_sm = 132;
    float* d_seg_v = nullptr; float4* d_seg_xys = nullptr; int* d_seg_counts = nullptr;
    unsigned *d_keys_a = nullptr, *d_vals_a = nullptr, *d_keys_b = nullptr, *d_vals_b = nullptr;
    int* d_seed_f = nullptr; float4* d_seed_vxys = nullptr; int* d_n_seeds = nullptr;
    float* d_lists = nullptr; int* d_list_counts = nullptr;
    unsigned char* d_occ = nullptr; size_t occ_bytes = 0;
    Joint* d_anns = nullptr; long long* d_ann_ids = nullptr; int* d_n_anns = nullptr; int* d_flags = nullptr;
    long long* d_grow_dbg = nullptr;      // k_grow diagnostics (rounds, picks, clocks per phase), [B][6]
    float4* d_out_ann = nullptr; long long* d_out_ids = nullptr; int* d_out_counts = nullptr;
    // packed results, double buffered (device + pinned host + event) so that a fetch can overlap the next decode
    unsigned char* d_result[2] = {nullptr, nullptr};
    unsigned char* h_result[2] = {nullptr, nullptr};
    cudaEvent_t ev_result[2] = {nullptr, nullptr};
    size_t result_bytes = 0, prefix_bytes = 0;
    int cur_result = 0;          // buffer the next decode writes
    int n_begun = 0, n_ended = 0;   // fetch_begin / fetch_end counters (at most 2 outstanding)
    int slot_batch[2] = {0, 0};
    // single-image host path
    float *d_in_cif = nullptr, *d_in_caf = nullptr, *d_in_init = nullptr; long long* d_in_init_ids = nullptr;
    int* d_in_init_count = nullptr; int in_init_cap = 0;
    // pinned staging
    cudaStream_t own_stream = nullptr;
    float defer_radius = 6.0f;        // PIFPAF_GROW_DEFER (a performance heuristic of k_grow, never changes results)
    GrowLayout grow{};                // warps (annotations in flight) per image and shared-memory plan of k_grow
    unsigned epoch = 1;               // occupancy tags: epoch (seed loop), epoch+1 (NMS)
    Dims last{};
    bool has_last = false;
    double last_revision = 1.0;
};

namespace {

int validate_dims(pifpaf_decoder* dec, int batch, int h, int w, int cif_stride, int caf_stride) {
    PIFPAF_CHECK_ARG(dec != nullptr, "decoder handle is null");
    PIFPAF_CHECK_ARG(batch >= 1 && batch <= dec->max_batch, "batch exceeds max_batch given at create()");
    PIFPAF_CHECK_ARG(h >= 1 && w >= 1 && h <= dec->max_h && w <= dec->max_w, "field shape exceeds max_h/max_w");
    PIFPAF_CHECK_ARG(cif_stride >= 1 && cif_stride <= dec->max_stride, "cif_stride exceeds max_stride");
    PIFPAF_CHECK_ARG(caf_stride >= 1 && caf_stride <= dec->max_stride, "caf_stride exceeds max_stride");
    return PIFPAF_OK;
}

Dims make_dims(const pifpaf_decoder* dec, int batch, int h, int w, int cif_stride, int caf_stride,
               double occ_reduction) {
    Dims d;
    d.B = batch; d.F = dec->F; d.C = dec->C; d.K = dec->K;
    d.h = h; d.w = w; d.hw = h * w;
    d.cif_stride = cif_stride; d.caf_stride = caf_stride;
    d.H = (h - 1) * cif_stride + 1; d.W = (w - 1) * cif_stride + 1;     // src/cif_hr.cpp:110-114
    d.Wp = (d.W + TILE - 1) / TILE * TILE;
    d.Ho = (int)((double)d.H / occ_reduction) + 1;                      // src/occupancy.cpp:47-48
    d.Wo = (int)((double)d.W / occ_reduction) + 1;
    d.tiles_x = d.Wp / TILE; d.tiles_y = (d.H + TILE - 1) / TILE;
    d.max_ann = dec->max_ann;
    return d;
}

}  // namespace

extern "C" {

int pifpaf_decoder_default_params(pifpaf_decoder_params_t* p) {
    PIFPAF_CHECK_ARG(p != nullptr, "params is null");
    std::memset(p, 0, sizeof(*p));
    p->cifhr_neighbors = 16; p->cifhr_threshold = 0.3;
    p->seed_threshold = 0.2;
    p->caf_score_th = 0.3; p->caf_cif_floor = 0.1;
    p->keypoint_threshold = 0.15; p->keypoint_threshold_rel = 0.5;
    p->reverse_match = 1; p->force_complete_caf_th = 0.001;
    p->nms_suppression = 0.00001; p->nms_instance_threshold = 0.15; p->nms_keypoint_threshold = 0.15;
    p->occ_reduction = 2.0; p->occ_min_scale = 4.0;
    p->cifhr_revision = 1.0;
    return PIFPAF_OK;
}

void pifpaf_decoder_destroy(pifpaf_decoder_t* dec) {
    if (!dec) return;
    cudaSetDevice(dec->device);
    void* dev_ptrs[] = {dec->d_skeleton, dec->d_adj_start, dec->d_adj_edge, dec->d_edge_lookup, dec->d_pair_id,
        dec->d_cifhr, dec->d_cells, dec->d_boxes, dec->d_cell_counts, dec->d_tile_epoch, dec->d_worklist,
        dec->d_work_count, dec->d_seg_v, dec->d_seg_xys,
        dec->d_seg_counts, dec->d_keys_a, dec->d_vals_a, dec->d_keys_b, dec->d_vals_b, dec->d_seed_f,
        dec->d_seed_vxys, dec->d_n_seeds, dec->d_lists, dec->d_list_counts, dec->d_occ, dec->d_anns,
        dec->d_ann_ids, dec->d_n_anns, dec->d_flags, dec->d_grow_dbg, dec->d_out_ann, dec->d_out_ids, dec->d_out_counts,
        dec->d_result[0], dec->d_result[1], dec->d_in_cif, dec->d_in_caf, dec->d_in_init,
        dec->d_in_init_ids, dec->d_in_init_count};
    for (void* p : dev_ptrs) if (p) cudaFree(p);
    for (int i = 0; i < 2; i++) {
        if (dec->h_result[i]) cudaFreeHost(dec->h_result[i]);
        if (dec->ev_result[i]) cudaEventDestroy(dec->ev_result[i]);
    }
    if (dec->own_stream) cudaStreamDestroy(dec->own_stream);
    delete dec;
}

int pifpaf_decoder_create(pifpaf_decoder_t** out, int32_t device, int32_t n_keypoints, int32_t n_cif_fields,
                          int32_t n_connections, const int64_t* skeleton,
                          int32_t max_batch, int32_t max_h, int32_t max_w, int32_t max_stride,
                          int32_t max_annotations) {
    PIFPAF_CHECK_ARG(out != nullptr, "out is null");
    *out = nullptr;
    PIFPAF_CHECK_ARG(n_keypoints >= 1 && n_cif_fields >= 1 && n_connections >= 0, "bad keypoint/field/connection count");
    PIFPAF_CHECK_ARG(n_cif_fields <= n_keypoints,
                     "NMS occupancy map must be of same size or smaller as annotation");   // src/nms_keypoints.cpp:30-31
    PIFPAF_CHECK_ARG(skeleton != nullptr || n_connections == 0, "skeleton is null");
    PIFPAF_CHECK_ARG(max_batch >= 1 && max_h >= 1 && max_w >= 1 && max_stride >= 1, "bad capacity");
    PIFPAF_CHECK_ARG(max_annotations >= 1 && max_annotations <= 8192, "max_annotations must be in [1, 8192]");
    PIFPAF_CHECK_ARG(n_connections <= (1 << 20), "too many connections");
    for (int c = 0; c < n_connections; c++) {
        PIFPAF_CHECK_ARG(skeleton[2 * c] >= 0 && skeleton[2 * c] < n_keypoints &&
                         skeleton[2 * c + 1] >= 0 && skeleton[2 * c + 1] < n_keypoints,
                         "skeleton index out of range (must be 0-based and < n_keypoints)");
    }
    int n_dev = 0;
    PIFPAF_CUDA_TRY(cudaGetDeviceCount(&n_dev));
    PIFPAF_CHECK_ARG(device >= 0 && device < n_dev, "no such CUDA device");
    PIFPAF_CUDA_TRY(cudaSetDevice(device));

    pifpaf_decoder* dec = new pifpaf_decoder();
    dec->device = device;
    dec->K = n_keypoints; dec->F = n_cif_fields; dec->C = n_connections;
    dec->max_batch = max_batch; dec->max_h = max_h; dec->max_w = max_w; dec->max_stride = max_stride;
    dec->max_ann = max_annotations;
    dec->skeleton.assign(skeleton, skeleton + 2 * (size_t)n_connections);

    const int K = dec->K, C = dec->C, F = dec->F;
    // graph tables -------------------------------------------------------
    std::vector<int> sk(2 * (size_t)C + 2, 0);
    for (int i = 0; i < 2 * C; i++) sk[i] = (int)skeleton[i];
    std::vector<int> adj_start(K + 1, 0), adj_edge;
    for (int j = 0; j < K; j++) {
        adj_start[j] = (int)adj_edge.size();
        for (int c = 0; c < C; c++) {           // src/cifcaf.cpp:323-345: first branch wins
            if (sk[2 * c] == j) adj_edge.push_back(2 * c);
            else if (sk[2 * c + 1] == j) adj_edge.push_back(2 * c + 1);
        }
    }
    adj_start[K] = (int)adj_edge.size();
    std::vector<int> edge_lookup(2 * (size_t)C + 2, 0), pair_id(2 * (size_t)C + 2, 0);
    for (int e = 0; e < 2 * C; e++) {
        const int c = e >> 1, dir = e & 1;
        const int start_i = sk[2 * c + dir], end_i = sk[2 * c + 1 - dir];
        int caf_i = 0, forward = 1;
        for (int f = 0; f < C; f++) {           // src/cifcaf.cpp:360-373
            if (sk[2 * f] == start_i && sk[2 * f + 1] == end_i) { forward = 1; break; }
            if (sk[2 * f + 1] == start_i && sk[2 * f] == end_i) { forward = 0; break; }
            caf_i++;
        }
        edge_lookup[e] = caf_i * 2 + forward;
        int pid = e;
        for (int e2 = 0; e2 < e; e2++) {
            const int c2 = e2 >> 1, d2 = e2 & 1;
            if (sk[2 * c2 + d2] == start_i && sk[2 * c2 + 1 - d2] == end_i) { pid = e2; break; }
        }
        pair_id[e] = pid;
    }
    if (adj_edge.empty()) adj_edge.push_back(0);

    int rc = PIFPAF_OK;
#define ALLOC(ptr, n) do { rc = dev_alloc(&(ptr), (n)); if (rc != PIFPAF_OK) { pifpaf_decoder_destroy(dec); return rc; } } while (0)
#define TRY_D(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { pifpaf::set_error("%s failed: %s", #expr, cudaGetErrorString(e__)); pifpaf_decoder_destroy(dec); return PIFPAF_E_CUDA; } } while (0)
    ALLOC(dec->d_skeleton, sk.size()); ALLOC(dec->d_adj_start, adj_start.size());
    ALLOC(dec->d_adj_edge, adj_edge.size()); ALLOC(dec->d_edge_lookup, edge_lookup.size());
    ALLOC(dec->d_pair_id, pair_id.size());
    TRY_D(cudaMemcpy(dec->d_skeleton, sk.data(), sizeof(int) * sk.size(), cudaMemcpyHostToDevice));
    TRY_D(cudaMemcpy(dec->d_adj_start, adj_start.data(), sizeof(int) * adj_start.size(), cudaMemcpyHostToDevice));
    TRY_D(cudaMemcpy(dec->d_adj_edge, adj_edge.data(), sizeof(int) * adj_edge.size(), cudaMemcpyHostToDevice));
    TRY_D(cudaMemcpy(dec->d_edge_lookup, edge_lookup.data(), sizeof(int) * edge_lookup.size(), cudaMemcpyHostToDevice));
    TRY_D(cudaMemcpy(dec->d_pair_id, pair_id.data(), sizeof(int) * pair_id.size(), cudaMemcpyHostToDevice));

    // workspace ------------------------------------------------------------
    const size_t B = max_batch, hw = (size_t)max_h * max_w;
    const size_t Hm = (size_t)(max_h - 1) * max_stride + 1, Wm = (size_t)(max_w - 1) * max_stride + 1;
    const size_t Wpm = (Wm + TILE - 1) / TILE * TILE;
    ALLOC(dec->d_cifhr, B * F * Hm * Wpm);
    ALLOC(dec->d_cells, B * F * hw); ALLOC(dec->d_boxes, B * F * hw); ALLOC(dec->d_cell_counts, B * F);
    {
        const size_t tiles_max = (Wpm / TILE) * ((Hm + TILE - 1) / TILE);
        dec->tile_epoch_elems = B * F * tiles_max;
        ALLOC(dec->d_tile_epoch, dec->tile_epoch_elems); ALLOC(dec->d_worklist, dec->tile_epoch_elems);
        ALLOC(dec->d_work_count, 1);
        TRY_D(cudaMemset(dec->d_tile_epoch, 0, sizeof(unsigned) * dec->tile_epoch_elems));
        cudaDeviceProp prop;
        TRY_D(cudaGetDeviceProperties(&prop, device));
        dec->n_sm = prop.multiProcessorCount;
    }
    ALLOC(dec->d_seg_v, B * F * hw); ALLOC(dec->d_seg_xys, B * F * hw); ALLOC(dec->d_seg_counts, B * F);
    ALLOC(dec->d_keys_a, B * F * hw); ALLOC(dec->d_vals_a, B * F * hw);
    ALLOC(dec->d_keys_b, B * F * hw); ALLOC(dec->d_vals_b, B * F * hw);
    ALLOC(dec->d_seed_f, B * F * hw); ALLOC(dec->d_seed_vxys, B * F * hw); ALLOC(dec->d_n_seeds, B);
    ALLOC(dec->d_lists, B * (size_t)C * 2 * 7 * hw); ALLOC(dec->d_list_counts, B * (size_t)C * 2);
    // occupancy never needs more than the un-reduced map (reduction >= 1)
    dec->occ_bytes = B * F * (Hm + 1) * (Wm + 1);
    ALLOC(dec->d_occ, dec->occ_bytes);
    TRY_D(cudaMemset(dec->d_occ, 0, dec->occ_bytes));
    const size_t A = max_annotations;
    ALLOC(dec->d_anns, B * A * K); ALLOC(dec->d_ann_ids, B * A); ALLOC(dec->d_n_anns, B); ALLOC(dec->d_flags, B);
    ALLOC(dec->d_grow_dbg, B * 6);
    ALLOC(dec->d_out_ann, B * A * K); ALLOC(dec->d_out_ids, B * A); ALLOC(dec->d_out_counts, B);
    dec->result_bytes = result_header_bytes((int)B) + B * A * (K + 1) * sizeof(float4);
    // one async D2H copies the header and this much payload; the (rare) rest is fetched on demand
    dec->prefix_bytes = std::min(dec->result_bytes, result_header_bytes((int)B) + (size_t)512 * 1024);
    for (int i = 0; i < 2; i++) {
        ALLOC(dec->d_result[i], dec->result_bytes);
        TRY_D(cudaMallocHost(reinterpret_cast<void**>(&dec->h_result[i]), dec->result_bytes));
        TRY_D(cudaEventCreateWithFlags(&dec->ev_result[i], cudaEventDisableTiming));
    }
    ALLOC(dec->d_in_cif, (size_t)F * 5 * hw); ALLOC(dec->d_in_caf, (size_t)C * 8 * hw);
    dec->in_init_cap = max_annotations;
    ALLOC(dec->d_in_init, A * K * 4); ALLOC(dec->d_in_init_ids, A); ALLOC(dec->d_in_init_count, 1);
    TRY_D(cudaStreamCreateWithFlags(&dec->own_stream, cudaStreamNonBlocking));

    dec->grow = plan_grow(K, C);
    if (const char* e = std::getenv("PIFPAF_GROW_DEFER")) dec->defer_radius = (float)std::atof(e);
    TRY_D(raise_smem_limit((const void*)k_grow, device, dec->grow.smem));
    TRY_D(raise_smem_limit((const void*)k_force_complete, device, dec->grow.smem));
    const size_t ns = (sizeof(double) + 2 * sizeof(int)) * A + 16;
    TRY_D(raise_smem_limit((const void*)k_nms, device, ns));
    const size_t ss = sizeof(int) * (((size_t)F + 1 + 3) / 4 * 4 + 256 + 256 + 8) + 2 * 32 * 256 + 16;
    TRY_D(raise_smem_limit((const void*)k_seed_sort, device, ss));
    // the memsets / table uploads above ran on the legacy default stream; decodes are enqueued on caller streams
    // (possibly non-blocking ones) that do not order themselves behind it
    TRY_D(cudaDeviceSynchronize());
#undef ALLOC
#undef TRY_D
    *out = dec;
    return PIFPAF_OK;
}

int pifpaf_decoder_decode_device(pifpaf_decoder_t* dec, const float* cif_dev, const float* caf_dev,
                                 int32_t batch, int32_t h, int32_t w, int32_t cif_stride, int32_t caf_stride,
                                 const float* init_ann_dev, const int64_t* init_ids_dev,
                                 const int32_t* init_counts_dev, int32_t init_cap,
                                 const pifpaf_decoder_params_t* params, void* stream_v) {
    int rc = validate_dims(dec, batch, h, w, cif_stride, caf_stride);
    if (rc != PIFPAF_OK) return rc;
    PIFPAF_CHECK_ARG(cif_dev != nullptr && caf_dev != nullptr, "field pointer is null");
    PIFPAF_CHECK_ARG(params != nullptr, "params is null");
    PIFPAF_CHECK_ARG(params->occ_reduction >= 1.0, "occ_reduction must be >= 1");
    PIFPAF_CHECK_ARG(params->cifhr_neighbors != 0, "cifhr_neighbors must be non-zero");
    PIFPAF_CHECK_ARG(init_ann_dev == nullptr || (init_ids_dev != nullptr && init_counts_dev != nullptr),
                     "require initial_ids when initial_annotations are given");   // src/cifcaf.cpp:178
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    const pifpaf_decoder_params_t& p = *params;
    const Dims d = make_dims(dec, batch, h, w, cif_stride, caf_stride, p.occ_reduction);
    dec->last = d; dec->has_last = true; dec->last_revision = p.cifhr_revision;

    // occupancy epoch tags (Occupancy::clear == revision++, src/occupancy.cpp:71-77)
    if (dec->epoch + 1 > 254) {
        PIFPAF_CUDA_TRY(cudaMemsetAsync(dec->d_occ, 0, dec->occ_bytes, st));
        dec->epoch = 1;
    }
    const unsigned char tag_seed = (unsigned char)dec->epoch, tag_nms = (unsigned char)(dec->epoch + 1);
    dec->epoch += 2;

    GrowParams gp;
    gp.keypoint_threshold = p.keypoint_threshold; gp.keypoint_threshold_rel = p.keypoint_threshold_rel;
    gp.reverse_match = p.reverse_match; gp.greedy = p.greedy;
    gp.occ_reduction = p.occ_reduction; gp.occ_min_scale_reduced = p.occ_min_scale / p.occ_reduction;
    gp.nms_suppression = p.nms_suppression; gp.nms_instance_threshold = p.nms_instance_threshold;
    gp.nms_keypoint_threshold = p.nms_keypoint_threshold;
    gp.defer_radius = dec->defer_radius;
    Graph gr{dec->d_skeleton, dec->d_adj_start, dec->d_adj_edge, dec->d_edge_lookup, dec->d_pair_id};

    // CifHr (src/cifcaf.cpp:140-142: accumulate(cif, stride, min_scale 0.0, factor 1.0)).  A new epoch
    // invalidates every tile (== the fresh zeroed buffer of a new reference instance) without touching memory.
    if (++dec->hr_epoch == 0) {
        PIFPAF_CUDA_TRY(cudaMemsetAsync(dec->d_tile_epoch, 0, sizeof(unsigned) * dec->tile_epoch_elems, st));
        dec->hr_epoch = 1;
    }
    const unsigned hr_epoch = dec->hr_epoch;
    if (!p.cifhr_ablation_skip) {
        const float min_scale_f = (float)(0.0 / (double)cif_stride);
        PIFPAF_CUDA_TRY(cudaMemsetAsync(dec->d_work_count, 0, sizeof(int), st));
        k_cif_compact<<<dim3(d.F, d.B), NT, 0, st>>>(cif_dev, d, 0, p.cifhr_threshold, (long long)p.cifhr_neighbors,
                                                     min_scale_f, 1.0, dec->d_cells, dec->d_boxes, dec->d_cell_counts,
                                                     dec->d_tile_epoch, hr_epoch, dec->d_worklist, dec->d_work_count);
        PIFPAF_LAUNCH_CHECK();
        k_cifhr_tiles<<<dec->n_sm * 8, NT, 0, st>>>(d, p.cifhr_revision, dec->d_cells, dec->d_boxes,
                                                    dec->d_cell_counts, dec->d_worklist, dec->d_work_count, dec->d_cifhr);
        PIFPAF_LAUNCH_CHECK();
    }
    // seeds (src/cifcaf.cpp:144-148)
    k_seed_candidates<<<dim3(d.F, d.B), NT, 0, st>>>(cif_dev, d, dec->d_cifhr, dec->d_tile_epoch, hr_epoch,
                                                     p.cifhr_revision, p.seed_threshold,
                                                     p.seeds_ablation_nms, p.seeds_ablation_no_rescore, 0,
                                                     dec->d_seg_v, dec->d_seg_xys, dec->d_seg_counts);
    PIFPAF_LAUNCH_CHECK();
    const size_t ss = sizeof(int) * (((size_t)d.F + 1 + 3) / 4 * 4 + 256 + 256 + 8) + 2 * 32 * 256 + 16;
    k_seed_sort<<<d.B, SORT_NT, ss, st>>>(d, dec->d_seg_counts, dec->d_seg_v, dec->d_seg_xys, dec->d_keys_a,
                                          dec->d_vals_a, dec->d_keys_b, dec->d_vals_b, dec->d_seed_f,
                                          dec->d_seed_vxys, nullptr, dec->d_n_seeds);
    PIFPAF_LAUNCH_CHECK();
    // caf scored (src/cifcaf.cpp:153-161: CafScored(cifhr, rev, -1.0, 0.1))
    if (d.C > 0) {
        k_caf_scored<<<dim3(d.C, d.B), NT, 0, st>>>(caf_dev, d, dec->d_skeleton, dec->d_cifhr, dec->d_tile_epoch,
                                                    hr_epoch, p.cifhr_revision, p.caf_score_th, p.caf_cif_floor, p.caf_ablation_no_rescore,
                                                    dec->d_lists, dec->d_list_counts);
        PIFPAF_LAUNCH_CHECK();
    }
    const size_t gs = dec->grow.smem;
    const int grow_threads = 32 * dec->grow.workers;
    k_grow<<<d.B, grow_threads, gs, st>>>(d, gr, gp, dec->grow.list_cap, dec->grow.ext_cap, dec->d_seed_f, dec->d_seed_vxys, dec->d_n_seeds, dec->d_lists,
                                dec->d_list_counts, dec->d_occ, tag_seed, init_ann_dev,
                                reinterpret_cast<const long long*>(init_ids_dev), init_counts_dev, init_cap,
                                dec->d_anns, dec->d_ann_ids, dec->d_n_anns, dec->d_flags, dec->d_grow_dbg);
    PIFPAF_LAUNCH_CHECK();
    if (p.force_complete && d.C > 0) {
        // src/cifcaf.cpp:414-426: CafScored(cifhr, rev, force_complete_caf_th, 0.1); score_th_ >= 0 ? it : default
        const double th = p.force_complete_caf_th >= 0.0 ? p.force_complete_caf_th : p.caf_score_th;
        k_caf_scored<<<dim3(d.C, d.B), NT, 0, st>>>(caf_dev, d, dec->d_skeleton, dec->d_cifhr, dec->d_tile_epoch,
                                                    hr_epoch, p.cifhr_revision, th, 0.1, p.caf_ablation_no_rescore, dec->d_lists, dec->d_list_counts);
        PIFPAF_LAUNCH_CHECK();
        k_force_complete<<<d.B, grow_threads, gs, st>>>(d, gr, gp, dec->grow.list_cap, dec->grow.ext_cap, dec->d_lists, dec->d_list_counts, dec->d_anns, dec->d_n_anns);
        PIFPAF_LAUNCH_CHECK();
    }
    const size_t ns = (sizeof(double) + 2 * sizeof(int)) * (size_t)d.max_ann + 16;
    k_nms<<<d.B, NT, ns, st>>>(d, gp, dec->d_anns, dec->d_ann_ids, dec->d_n_anns, dec->d_occ, tag_nms,
                               dec->d_out_ann, dec->d_out_ids, dec->d_out_counts);
    PIFPAF_LAUNCH_CHECK();
    k_pack<<<d.B, NT, 0, st>>>(d, dec->d_out_ann, dec->d_out_ids, dec->d_out_counts, dec->d_flags,
                               dec->d_result[dec->cur_result]);
    PIFPAF_LAUNCH_CHECK();
    return PIFPAF_OK;
}

int pifpaf_decoder_fetch_begin(pifpaf_decoder_t* dec, void* stream_v) {
    PIFPAF_CHECK_ARG(dec != nullptr && dec->has_last, "no decode to fetch");
    PIFPAF_CHECK_ARG(dec->n_begun - dec->n_ended < 2, "at most two fetches may be outstanding");
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    const int slot = dec->cur_result;
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(dec->h_result[slot], dec->d_result[slot], dec->prefix_bytes,
                                    cudaMemcpyDeviceToHost, st));
    PIFPAF_CUDA_TRY(cudaEventRecord(dec->ev_result[slot], st));
    dec->slot_batch[slot] = dec->last.B;
    dec->cur_result ^= 1;          // the next decode packs into the other buffer
    dec->n_begun++;
    return PIFPAF_OK;
}

int pifpaf_decoder_fetch_peek(pifpaf_decoder_t* dec, int32_t* counts) {
    PIFPAF_CHECK_ARG(dec != nullptr && dec->n_begun > dec->n_ended, "fetch_peek without fetch_begin");
    PIFPAF_CHECK_ARG(counts != nullptr, "counts is null");
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    const int outstanding = dec->n_begun - dec->n_ended;
    const int slot = (outstanding == 2) ? dec->cur_result : (dec->cur_result ^ 1);
    PIFPAF_CUDA_TRY(cudaEventSynchronize(dec->ev_result[slot]));
    const int* hdr = reinterpret_cast<const int*>(dec->h_result[slot]);
    for (int b = 0; b < dec->slot_batch[slot]; b++) counts[b] = hdr[b];
    return PIFPAF_OK;
}

int pifpaf_decoder_fetch_end(pifpaf_decoder_t* dec, int32_t* counts, float* ann, int64_t* ids, int32_t ann_cap) {
    PIFPAF_CHECK_ARG(dec != nullptr && dec->n_begun > dec->n_ended, "fetch_end without fetch_begin");
    PIFPAF_CHECK_ARG(counts != nullptr, "counts is null");
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    // oldest outstanding slot: slots alternate, so it is cur_result when two are outstanding, else the other one
    const int outstanding = dec->n_begun - dec->n_ended;
    const int slot = (outstanding == 2) ? dec->cur_result : (dec->cur_result ^ 1);
    PIFPAF_CUDA_TRY(cudaEventSynchronize(dec->ev_result[slot]));
    dec->n_ended++;
    const int B = dec->slot_batch[slot], K = dec->K;
    const int* hdr = reinterpret_cast<const int*>(dec->h_result[slot]);
    const int* h_counts = hdr; const int* h_flags = hdr + B; const int* h_off = hdr + 2 * B;
    const int total = h_off[B];
    const size_t hb = result_header_bytes(B), rec_bytes = (size_t)(K + 1) * sizeof(float4);
    const size_t need = hb + (size_t)total * rec_bytes;
    if (need > dec->prefix_bytes && ann != nullptr) {
        PIFPAF_CUDA_TRY(cudaMemcpyAsync(dec->h_result[slot] + dec->prefix_bytes, dec->d_result[slot] + dec->prefix_bytes,
                                        need - dec->prefix_bytes, cudaMemcpyDeviceToHost, dec->own_stream));
        PIFPAF_CUDA_TRY(cudaStreamSynchronize(dec->own_stream));
    }
    const unsigned char* recs = dec->h_result[slot] + hb;
    bool overflow = false;
    for (int b = 0; b < B; b++) {
        counts[b] = h_counts[b];
        if (h_flags[b]) overflow = true;
        if (ann == nullptr) continue;
        int n = h_counts[b];
        if (n > ann_cap) { overflow = true; n = ann_cap; }
        for (int a = 0; a < n; a++) {
            const unsigned char* r = recs + (size_t)(h_off[b] + a) * rec_bytes;
            std::memcpy(ann + ((size_t)b * ann_cap + a) * K * 4, r, sizeof(float) * 4 * (size_t)K);
            if (ids) std::memcpy(ids + (size_t)b * ann_cap + a, r + sizeof(float4) * (size_t)K, sizeof(int64_t));
        }
    }
    if (overflow) {
        pifpaf::set_error("annotation capacity exceeded (max_annotations=%d, ann_cap=%d): "
                          "create the decoder with a larger max_annotations", dec->max_ann, ann_cap);
        return PIFPAF_E_OVERFLOW;
    }
    return PIFPAF_OK;
}

int pifpaf_decoder_fetch(pifpaf_decoder_t* dec, int32_t* counts, float* ann, int64_t* ids,
                         int32_t ann_cap, void* stream_v) {
    int rc = pifpaf_decoder_fetch_begin(dec, stream_v);
    if (rc != PIFPAF_OK) return rc;
    return pifpaf_decoder_fetch_end(dec, counts, ann, ids, ann_cap);
}

int pifpaf_decoder_call(pifpaf_decoder_t* dec, const float* cif, int32_t cif_stride,
                        const float* caf, int32_t caf_stride, int32_t h, int32_t w,
                        const float* initial_annotations, const int64_t* initial_ids, int32_t n_initial,
                        const pifpaf_decoder_params_t* params,
                        float* out_ann, int64_t* out_ids, int32_t cap, int32_t* n_out) {
    int rc = validate_dims(dec, 1, h, w, cif_stride, caf_stride);
    if (rc != PIFPAF_OK) return rc;
    PIFPAF_CHECK_ARG(cif != nullptr && caf != nullptr, "cif_field / caf_field is null");
    PIFPAF_CHECK_ARG(n_out != nullptr, "n_out is null");
    PIFPAF_CHECK_ARG(n_initial >= 0 && n_initial <= dec->in_init_cap, "too many initial annotations");
    PIFPAF_CHECK_ARG(n_initial == 0 || (initial_annotations != nullptr && initial_ids != nullptr),
                     "require initial_ids when initial_annotations are given");
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    cudaStream_t st = dec->own_stream;
    const size_t hw = (size_t)h * w;
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(dec->d_in_cif, cif, sizeof(float) * dec->F * 5 * hw, cudaMemcpyHostToDevice, st));
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(dec->d_in_caf, caf, sizeof(float) * dec->C * 8 * hw, cudaMemcpyHostToDevice, st));
    const float* d_init = nullptr; const int64_t* d_ids = nullptr; const int* d_cnt = nullptr;
    if (n_initial > 0) {
        PIFPAF_CUDA_TRY(cudaMemcpyAsync(dec->d_in_init, initial_annotations, sizeof(float) * 4 * (size_t)n_initial * dec->K,
                                        cudaMemcpyHostToDevice, st));
        PIFPAF_CUDA_TRY(cudaMemcpyAsync(dec->d_in_init_ids, initial_ids, sizeof(int64_t) * (size_t)n_initial,
                                        cudaMemcpyHostToDevice, st));
        PIFPAF_CUDA_TRY(cudaMemcpyAsync(dec->d_in_init_count, &n_initial, sizeof(int), cudaMemcpyHostToDevice, st));
        d_init = dec->d_in_init; d_ids = reinterpret_cast<const int64_t*>(dec->d_in_init_ids); d_cnt = dec->d_in_init_count;
    }
    rc = pifpaf_decoder_decode_device(dec, dec->d_in_cif, dec->d_in_caf, 1, h, w, cif_stride, caf_stride,
                                      d_init, d_ids, d_cnt, dec->in_init_cap, params, st);
    if (rc != PIFPAF_OK) return rc;
    int32_t count = 0;
    rc = pifpaf_decoder_fetch(dec, &count, out_ann, out_ids, cap, st);
    *n_out = count;
    return rc;
}

int pifpaf_decoder_tap_cifhr(pifpaf_decoder_t* dec, int32_t b, float* out, int64_t out_elems) {
    PIFPAF_CHECK_ARG(dec != nullptr && dec->has_last, "no decode to tap");
    const Dims& d = dec->last;
    PIFPAF_CHECK_ARG(b >= 0 && b < d.B, "image index out of range");
    PIFPAF_CHECK_ARG(out != nullptr && out_elems >= (int64_t)d.F * d.H * d.W, "output buffer too small");
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    PIFPAF_CUDA_TRY(cudaDeviceSynchronize());
    k_cifhr_materialize<<<dim3(d.tiles_x * d.tiles_y, d.F), NT>>>(d, b, dec->d_tile_epoch, dec->hr_epoch, dec->d_cifhr);
    PIFPAF_LAUNCH_CHECK();
    PIFPAF_CUDA_TRY(cudaDeviceSynchronize());
    PIFPAF_CUDA_TRY(cudaMemcpy2D(out, sizeof(float) * d.W, dec->d_cifhr + (size_t)b * d.F * d.H * d.Wp,
                                 sizeof(float) * d.Wp, sizeof(float) * d.W, (size_t)d.F * d.H, cudaMemcpyDeviceToHost));
    return PIFPAF_OK;
}

int pifpaf_decoder_tap_seeds(pifpaf_decoder_t* dec, int32_t b, int64_t* out_f, float* out_vxys,
                             int64_t cap, int64_t* n_out) {
    PIFPAF_CHECK_ARG(dec != nullptr && dec->has_last, "no decode to tap");
    const Dims& d = dec->last;
    PIFPAF_CHECK_ARG(b >= 0 && b < d.B && n_out != nullptr, "bad argument");
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    PIFPAF_CUDA_TRY(cudaDeviceSynchronize());
    int n = 0;
    PIFPAF_CUDA_TRY(cudaMemcpy(&n, dec->d_n_seeds + b, sizeof(int), cudaMemcpyDeviceToHost));
    *n_out = n;
    const int m = (int)std::min<int64_t>(n, cap);
    if (m > 0 && out_f != nullptr && out_vxys != nullptr) {
        std::vector<int> f(m);
        const size_t img = (size_t)b * d.F * d.hw;
        PIFPAF_CUDA_TRY(cudaMemcpy(f.data(), dec->d_seed_f + img, sizeof(int) * m, cudaMemcpyDeviceToHost));
        PIFPAF_CUDA_TRY(cudaMemcpy(out_vxys, dec->d_seed_vxys + img, sizeof(float4) * m, cudaMemcpyDeviceToHost));
        for (int i = 0; i < m; i++) out_f[i] = f[i];
    }
    return PIFPAF_OK;
}

int pifpaf_decoder_tap_caf(pifpaf_decoder_t* dec, int32_t b, float* out_fwd, int64_t* n_fwd,
                           float* out_bwd, int64_t* n_bwd) {
    PIFPAF_CHECK_ARG(dec != nullptr && dec->has_last, "no decode to tap");
    const Dims& d = dec->last;
    PIFPAF_CHECK_ARG(b >= 0 && b < d.B, "image index out of range");
    PIFPAF_CHECK_ARG(out_fwd && n_fwd && out_bwd && n_bwd, "output pointer is null");
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    PIFPAF_CUDA_TRY(cudaDeviceSynchronize());
    std::vector<float> soa((size_t)d.C * 2 * 7 * d.hw);
    std::vector<int> cnt((size_t)d.C * 2);
    if (d.C == 0) return PIFPAF_OK;
    PIFPAF_CUDA_TRY(cudaMemcpy(soa.data(), dec->d_lists + (size_t)b * d.C * 2 * 7 * d.hw, sizeof(float) * soa.size(),
                               cudaMemcpyDeviceToHost));
    PIFPAF_CUDA_TRY(cudaMemcpy(cnt.data(), dec->d_list_counts + (size_t)b * d.C * 2, sizeof(int) * cnt.size(),
                               cudaMemcpyDeviceToHost));
    for (int c = 0; c < d.C; c++) {
        for (int dir = 0; dir < 2; dir++) {
            const int n = cnt[c * 2 + dir];
            float* dst = (dir == 0 ? out_fwd : out_bwd) + (size_t)c * d.hw * 7;
            const float* src = soa.data() + ((size_t)(c * 2 + dir) * 7) * d.hw;
            for (int i = 0; i < n; i++)
                for (int k = 0; k < 7; k++) dst[(size_t)i * 7 + k] = src[(size_t)k * d.hw + i];
            (dir == 0 ? n_fwd : n_bwd)[c] = n;
        }
    }
    return PIFPAF_OK;
}

int pifpaf_decoder_debug_set_epochs(pifpaf_decoder_t* dec, uint32_t occupancy_epoch, uint32_t cifhr_epoch) {
    PIFPAF_CHECK_ARG(dec != nullptr, "decoder handle is null");
    PIFPAF_CHECK_ARG(occupancy_epoch >= 1 && occupancy_epoch <= 255 && (occupancy_epoch & 1u) == 1u,
                     "occupancy epoch must be odd and in [1, 255]");
    dec->epoch = occupancy_epoch;
    dec->hr_epoch = cifhr_epoch;
    return PIFPAF_OK;
}

int pifpaf_decoder_last_stats(pifpaf_decoder_t* dec, int64_t* stats, int32_t n_stats) {
    PIFPAF_CHECK_ARG(dec != nullptr && dec->has_last, "no decode to report on");
    PIFPAF_CHECK_ARG(stats != nullptr && n_stats >= 4, "stats must hold at least 4 values");
    const Dims& d = dec->last;
    PIFPAF_CUDA_TRY(cudaSetDevice(dec->device));
    PIFPAF_CUDA_TRY(cudaDeviceSynchronize());
    int tiles = 0;
    PIFPAF_CUDA_TRY(cudaMemcpy(&tiles, dec->d_work_count, sizeof(int), cudaMemcpyDeviceToHost));
    std::vector<int> seeds(d.B), anns(d.B), lists((size_t)d.B * d.C * 2 + 1);
    PIFPAF_CUDA_TRY(cudaMemcpy(seeds.data(), dec->d_n_seeds, sizeof(int) * d.B, cudaMemcpyDeviceToHost));
    PIFPAF_CUDA_TRY(cudaMemcpy(anns.data(), dec->d_n_anns, sizeof(int) * d.B, cudaMemcpyDeviceToHost));
    if (d.C > 0)
        PIFPAF_CUDA_TRY(cudaMemcpy(lists.data(), dec->d_list_counts, sizeof(int) * (size_t)d.B * d.C * 2, cudaMemcpyDeviceToHost));
    long long ns = 0, na = 0, nl = 0;
    for (int b = 0; b < d.B; b++) { ns += seeds[b]; na += anns[b]; }
    for (size_t i = 0; i < (size_t)d.B * d.C * 2; i++) nl += lists[i];
    stats[0] = (int64_t)tiles * TILE * TILE;   // hi-res CifHr pixels written (sparse map)
    stats[1] = ns; stats[2] = nl; stats[3] = na;
    if (n_stats >= 10) {       // k_grow diagnostics, summed over the batch: rounds, picks, clocks in init/select/grow/commit
        std::vector<long long> dbg((size_t)d.B * 6);
        PIFPAF_CUDA_TRY(cudaMemcpy(dbg.data(), dec->d_grow_dbg, sizeof(long long) * dbg.size(), cudaMemcpyDeviceToHost));
        for (int k = 0; k < 6; k++) { long long t = 0; for (int b = 0; b < d.B; b++) t += dbg[(size_t)b * 6 + k]; stats[4 + k] = t; }
    }
    return PIFPAF_OK;
}

int pifpaf_grow_connection_blend(const float* caf, int64_t n, double x, double y, double s,
                                 double filter_sigmas, int32_t only_max, double* out_xysv) {
    PIFPAF_CHECK_ARG(out_xysv != nullptr, "out is null");
    PIFPAF_CHECK_ARG(n >= 0 && n < (1 << 28), "bad list length");
    PIFPAF_CHECK_ARG(caf != nullptr || n == 0, "caf is null");
    float* d_l = nullptr; double* d_o = nullptr;
    std::vector<float> soa((size_t)7 * (n ? n : 1));
    for (int64_t i = 0; i < n; i++)
        for (int k = 0; k < 7; k++) soa[(size_t)k * n + i] = caf[(size_t)i * 7 + k];
    PIFPAF_CUDA_TRY(cudaMalloc(reinterpret_cast<void**>(&d_l), sizeof(float) * soa.size()));
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&d_o), sizeof(double) * 4);
    if (e != cudaSuccess) { cudaFree(d_l); pifpaf::set_error("cudaMalloc failed"); return PIFPAF_E_CUDA; }
    cudaMemcpy(d_l, soa.data(), sizeof(float) * soa.size(), cudaMemcpyHostToDevice);
    k_blend_single<<<1, 32>>>(d_l, (int)n, x, y, s, filter_sigmas, only_max, d_o);
    pifpaf::count_launch();
    e = cudaMemcpy(out_xysv, d_o, sizeof(double) * 4, cudaMemcpyDeviceToHost);
    cudaFree(d_l); cudaFree(d_o);
    if (e != cudaSuccess) { pifpaf::set_error("grow_connection_blend failed: %s", cudaGetErrorString(e)); return PIFPAF_E_CUDA; }
    return PIFPAF_OK;
}

}  // extern "C"

// =====================================================================================================================
// CifDet decoder (SURVEY.md 8f rank 3).  Replaces torch.classes.openpifpaf_decoder.CifDet
// (csrc/src/cifdet.cpp:24-80, module.cpp:57-62) and, optionally, the torchvision NMS + score filter the reference's
// Python wrapper runs afterwards (decoder/cifdet.py:55-71).  CifDetHr / CifDetSeeds share the CIF kernels above
// (k_cif_compact / k_cifhr_tiles / k_seed_candidates / k_seed_sort in their det mode).
namespace {

constexpr int DET_REC = 8;     // floats per detection record: category, score, x1, y1, x2, y2, score after NMS, kept

// src/cifdet.cpp:50-66: walk the sorted seeds, keep those whose cell is free, mark 0.1 * min(w, h) around them.
// One warp per image: 32 seeds are tested against the map at once; the first free one (seed order) is accepted,
// marks the map, and the remaining lanes of the group are re-tested.
__global__ void __launch_bounds__(32) k_det_select(Dims d, GrowParams gp, int max_det,
                                                   const int* __restrict__ seed_f, const float4* __restrict__ seed_vxyw,
                                                   const float* __restrict__ seed_h, const int* __restrict__ n_seeds,
                                                   unsigned char* __restrict__ occ_map, unsigned char occ_tag,
                                                   float* __restrict__ records, int* __restrict__ counts) {
    const int b = blockIdx.x, lane = threadIdx.x;
    Occ occ;
    occ.map = occ_map + (size_t)b * d.F * d.Ho * d.Wo;
    occ.F = d.F; occ.Ho = d.Ho; occ.Wo = d.Wo;
    occ.reduction = gp.occ_reduction; occ.min_scale_reduced = gp.occ_min_scale_reduced;
    occ.tag = occ_tag;
    const size_t img = (size_t)b * d.F * d.hw;
    float* rec = records + (size_t)b * max_det * DET_REC;
    const int ns = n_seeds[b];
    int n_det = 0;
    for (int base = 0; base < ns && n_det < max_det; base += 32) {
        const int idx = base + lane;
        bool alive = idx < ns;
        int f = 0; float4 s = make_float4(0.f, 0.f, 0.f, 0.f); float bh = 0.f;
        if (alive) { f = seed_f[img + idx]; s = seed_vxyw[img + idx]; bh = seed_h[img + idx]; }
        while (n_det < max_det) {
            const bool is_free = alive && !occ_get(occ, f, (double)s.y, (double)s.z);
            const unsigned m = __ballot_sync(0xffffffffu, is_free);
            if (m == 0u) break;
            const int l = __ffs(m) - 1;
            const int fl = __shfl_sync(0xffffffffu, f, l);
            const float v = __shfl_sync(0xffffffffu, s.x, l), x = __shfl_sync(0xffffffffu, s.y, l);
            const float y = __shfl_sync(0xffffffffu, s.z, l), bw = __shfl_sync(0xffffffffu, s.w, l);
            const float hh = __shfl_sync(0xffffffffu, bh, l);
            occ_set_warp(occ, fl, (double)x, (double)y, 0.1 * (double)fminf(bw, hh), lane);
            __syncwarp();
            if (lane == 0) {
                float* r = rec + (size_t)n_det * DET_REC;
                r[0] = (float)(fl + 1); r[1] = v;
                r[2] = x - 0.5f * bw; r[3] = y - 0.5f * hh; r[4] = x + 0.5f * bw; r[5] = y + 0.5f * hh;
                r[6] = v; r[7] = 1.0f;
            }
            n_det++;
            alive = alive && lane > l;
        }
    }
    if (lane == 0) counts[b] = n_det;
}

// decoder/cifdet.py:55-64: torchvision.ops.batched_nms or torchvision.ops.nms, then scores *= suppression except for
// the kept ones, kept flag = score > instance_threshold.  torchvision's CPU kernel restated: stable descending order,
// IoU = inter / (area_i + area_j - inter) > threshold.
// batched_nms on CPU tensors dispatches on boxes.numel() > 4000 (torchvision/ops/boxes.py, batched_nms):
//   n <= 1000: _batched_nms_coordinate_trick, one nms over boxes shifted by category * (max coordinate + 1).  The
//              shift can overlap boxes of neighbouring categories (negative corners) and rounds shifted coordinates.
//   n > 1000:  _batched_nms_vanilla, one nms per category on the unshifted boxes.  Restated here as one pass over the
//              same stable order that compares only boxes of the same category: a category's subsequence of that
//              order is the order its own nms sorts into, and suppression never crosses categories.
constexpr int DET_NMS_VANILLA_MIN = 1001;
constexpr int DET_NMS_NT = 128;
__global__ void __launch_bounds__(DET_NMS_NT) k_det_nms(int max_det, float iou_threshold, int by_category,
                                                        float suppression, float instance_threshold,
                                                        float* __restrict__ records, const int* __restrict__ counts) {
    extern __shared__ __align__(16) unsigned char smem[];
    float4* box = reinterpret_cast<float4*>(smem);                    // [max_det] shifted boxes
    float* area = reinterpret_cast<float*>(box + max_det);            // [max_det]
    float* score = area + max_det;                                    // [max_det]
    int* order = reinterpret_cast<int*>(score + max_det);             // [max_det]
    unsigned char* sup = reinterpret_cast<unsigned char*>(order + max_det);   // [max_det]
    __shared__ float s_red[DET_NMS_NT / 32];
    __shared__ float s_max;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = counts[b];
    float* rec = records + (size_t)b * max_det * DET_REC;
    if (n == 0) return;
    float m = -INFINITY;
    for (int i = tid; i < n; i += DET_NMS_NT) {
        const float* r = rec + (size_t)i * DET_REC;
        m = fmaxf(m, fmaxf(fmaxf(r[2], r[3]), fmaxf(r[4], r[5])));
        score[i] = r[1];
        sup[i] = 0;
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) s_red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
        float mm = s_red[0];
        for (int i = 1; i < DET_NMS_NT / 32; i++) mm = fmaxf(mm, s_red[i]);
        s_max = mm;
    }
    __syncthreads();
    const float shift = s_max + 1.0f;                                  // max_coordinate + 1
    const bool per_category = by_category && n >= DET_NMS_VANILLA_MIN;
    const bool shifted = by_category && !per_category;
    for (int i = tid; i < n; i += DET_NMS_NT) {
        const float* r = rec + (size_t)i * DET_REC;
        const float off = shifted ? r[0] * shift : 0.0f;              // idxs.to(boxes) * (max_coordinate + 1)
        const float4 bx = make_float4(r[2] + off, r[3] + off, r[4] + off, r[5] + off);
        box[i] = bx;
        area[i] = (bx.z - bx.x) * (bx.w - bx.y);
        int rank = 0;                                                  // stable descending sort position
        for (int j = 0; j < n; j++) {
            const float sj = rec[(size_t)j * DET_REC + 1];
            if (sj > r[1] || (sj == r[1] && j < i)) rank++;
        }
        order[rank] = i;
    }
    __syncthreads();
    for (int oi = 0; oi < n; oi++) {
        const int i = order[oi];
        if (!sup[i]) {
            const float4 bi = box[i];
            const float ai = area[i];
            const float ci = per_category ? rec[(size_t)i * DET_REC] : 0.0f;
            for (int oj = oi + 1 + tid; oj < n; oj += DET_NMS_NT) {
                const int j = order[oj];
                if (sup[j]) continue;
                if (per_category && rec[(size_t)j * DET_REC] != ci) continue;
                const float4 bj = box[j];
                const float xx1 = fmaxf(bi.x, bj.x), yy1 = fmaxf(bi.y, bj.y);
                const float xx2 = fminf(bi.z, bj.z), yy2 = fminf(bi.w, bj.w);
                const float w = fmaxf(0.0f, xx2 - xx1), h = fmaxf(0.0f, yy2 - yy1);
                const float inter = w * h;
                const float ovr = inter / (ai + area[j] - inter);
                if (ovr > iou_threshold) sup[j] = 1;
            }
        }
        __syncthreads();
    }
    for (int i = tid; i < n; i += DET_NMS_NT) {
        float* r = rec + (size_t)i * DET_REC;
        const float sc = sup[i] ? score[i] * suppression : score[i];
        r[6] = sc;
        r[7] = sc > instance_threshold ? 1.0f : 0.0f;
    }
}

size_t det_nms_smem(int max_det) { return (size_t)max_det * (sizeof(float4) + 2 * sizeof(float) + sizeof(int) + 1) + 16; }

}  // namespace

struct pifpaf_cifdet {
    int device = 0, F = 0;
    int max_batch = 0, max_h = 0, max_w = 0, max_stride = 0, max_det = 0;
    int n_sm = 132;
    float* d_cifhr = nullptr;
    float4* d_cells = nullptr; int4* d_boxes = nullptr; int* d_cell_counts = nullptr;
    unsigned* d_tile_epoch = nullptr; int* d_worklist = nullptr; int* d_work_count = nullptr;
    unsigned hr_epoch = 0; size_t tile_epoch_elems = 0;
    float* d_seg_v = nullptr; float4* d_seg_xys = nullptr; int* d_seg_counts = nullptr;
    unsigned *d_keys_a = nullptr, *d_vals_a = nullptr, *d_keys_b = nullptr, *d_vals_b = nullptr;
    int* d_seed_f = nullptr; float4* d_seed_vxyw = nullptr; float* d_seed_h = nullptr; int* d_n_seeds = nullptr;
    unsigned char* d_occ = nullptr; size_t occ_bytes = 0; unsigned epoch = 1;
    float* d_records = nullptr; int* d_counts = nullptr;
    float* h_records = nullptr; int* h_counts = nullptr;       // pinned
    float* d_in_field = nullptr;
    cudaStream_t own_stream = nullptr;
    Dims last{}; bool has_last = false;
};

extern "C" {

int pifpaf_cifdet_default_params(pifpaf_cifdet_params_t* p) {
    PIFPAF_CHECK_ARG(p != nullptr, "params is null");
    std::memset(p, 0, sizeof(*p));
    p->cifhr_neighbors = 16; p->cifhr_threshold = 0.3;       // csrc/src/cif_hr.cpp:13-14
    p->seed_threshold = 0.2;                                  // CifDetSeeds::threshold, csrc/src/cif_seeds.cpp:12
    p->occ_reduction = 2.0; p->occ_min_scale = 4.0;           // include/openpifpaf/decoder/cifdet.hpp:40
    p->cifhr_revision = 1.0;
    p->max_detections_before_nms = 120;                       // csrc/src/cifdet.cpp:16
    p->nms = 0; p->nms_by_category = 1;
    p->iou_threshold = 0.5; p->suppression = 0.1; p->instance_threshold = 0.15;   // decoder/cifdet.py:17-21
    return PIFPAF_OK;
}

void pifpaf_cifdet_destroy(pifpaf_cifdet_t* det) {
    if (!det) return;
    cudaSetDevice(det->device);
    void* dev_ptrs[] = {det->d_cifhr, det->d_cells, det->d_boxes, det->d_cell_counts, det->d_tile_epoch, det->d_worklist,
        det->d_work_count, det->d_seg_v, det->d_seg_xys, det->d_seg_counts, det->d_keys_a, det->d_vals_a, det->d_keys_b,
        det->d_vals_b, det->d_seed_f, det->d_seed_vxyw, det->d_seed_h, det->d_n_seeds, det->d_occ, det->d_records,
        det->d_counts, det->d_in_field};
    for (void* p : dev_ptrs) if (p) cudaFree(p);
    if (det->h_records) cudaFreeHost(det->h_records);
    if (det->h_counts) cudaFreeHost(det->h_counts);
    if (det->own_stream) cudaStreamDestroy(det->own_stream);
    delete det;
}

int pifpaf_cifdet_create(pifpaf_cifdet_t** out, int32_t device, int32_t n_categories,
                         int32_t max_batch, int32_t max_h, int32_t max_w, int32_t max_stride, int32_t max_detections) {
    PIFPAF_CHECK_ARG(out != nullptr, "out is null");
    *out = nullptr;
    PIFPAF_CHECK_ARG(n_categories >= 1, "bad category count");
    PIFPAF_CHECK_ARG(max_batch >= 1 && max_h >= 1 && max_w >= 1 && max_stride >= 1, "bad capacity");
    PIFPAF_CHECK_ARG(max_detections >= 1 && max_detections <= 4096, "max_detections must be in [1, 4096]");
    int n_dev = 0;
    PIFPAF_CUDA_TRY(cudaGetDeviceCount(&n_dev));
    PIFPAF_CHECK_ARG(device >= 0 && device < n_dev, "no such CUDA device");
    PIFPAF_CUDA_TRY(cudaSetDevice(device));
    pifpaf_cifdet* det = new pifpaf_cifdet();
    det->device = device; det->F = n_categories;
    det->max_batch = max_batch; det->max_h = max_h; det->max_w = max_w; det->max_stride = max_stride;
    det->max_det = max_detections;
    int rc = PIFPAF_OK;
#define ALLOC(ptr, n) do { rc = dev_alloc(&(ptr), (n)); if (rc != PIFPAF_OK) { pifpaf_cifdet_destroy(det); return rc; } } while (0)
#define TRY_D(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { pifpaf::set_error("%s failed: %s", #expr, cudaGetErrorString(e__)); pifpaf_cifdet_destroy(det); return PIFPAF_E_CUDA; } } while (0)
    const size_t B = max_batch, F = n_categories, hw = (size_t)max_h * max_w;
    const size_t Hm = (size_t)(max_h - 1) * max_stride + 1, Wm = (size_t)(max_w - 1) * max_stride + 1;
    const size_t Wpm = (Wm + TILE - 1) / TILE * TILE;
    ALLOC(det->d_cifhr, B * F * Hm * Wpm);
    ALLOC(det->d_cells, B * F * hw); ALLOC(det->d_boxes, B * F * hw); ALLOC(det->d_cell_counts, B * F);
    const size_t tiles_max = (Wpm / TILE) * ((Hm + TILE - 1) / TILE);
    det->tile_epoch_elems = B * F * tiles_max;
    ALLOC(det->d_tile_epoch, det->tile_epoch_elems); ALLOC(det->d_worklist, det->tile_epoch_elems);
    ALLOC(det->d_work_count, 1);
    TRY_D(cudaMemset(det->d_tile_epoch, 0, sizeof(unsigned) * det->tile_epoch_elems));
    cudaDeviceProp prop;
    TRY_D(cudaGetDeviceProperties(&prop, device));
    det->n_sm = prop.multiProcessorCount;
    ALLOC(det->d_seg_v, B * F * hw); ALLOC(det->d_seg_xys, B * F * hw); ALLOC(det->d_seg_counts, B * F);
    ALLOC(det->d_keys_a, B * F * hw); ALLOC(det->d_vals_a, B * F * hw);
    ALLOC(det->d_keys_b, B * F * hw); ALLOC(det->d_vals_b, B * F * hw);
    ALLOC(det->d_seed_f, B * F * hw); ALLOC(det->d_seed_vxyw, B * F * hw); ALLOC(det->d_seed_h, B * F * hw);
    ALLOC(det->d_n_seeds, B);
    det->occ_bytes = B * F * (Hm + 1) * (Wm + 1);
    ALLOC(det->d_occ, det->occ_bytes);
    TRY_D(cudaMemset(det->d_occ, 0, det->occ_bytes));
    ALLOC(det->d_records, B * (size_t)max_detections * DET_REC); ALLOC(det->d_counts, B);
    TRY_D(cudaMallocHost(reinterpret_cast<void**>(&det->h_records), sizeof(float) * B * (size_t)max_detections * DET_REC));
    TRY_D(cudaMallocHost(reinterpret_cast<void**>(&det->h_counts), sizeof(int) * B));
    ALLOC(det->d_in_field, F * 6 * hw);
    TRY_D(cudaStreamCreateWithFlags(&det->own_stream, cudaStreamNonBlocking));
    const size_t ss = sizeof(int) * (((size_t)F + 1 + 3) / 4 * 4 + 256 + 256 + 8) + 2 * 32 * 256 + 16;
    TRY_D(raise_smem_limit((const void*)k_seed_sort, device, std::max(ss, (size_t)48 * 1024)));
    TRY_D(raise_smem_limit((const void*)k_det_nms, device, std::max(det_nms_smem(max_detections), (size_t)48 * 1024)));
    TRY_D(cudaDeviceSynchronize());
#undef ALLOC
#undef TRY_D
    *out = det;
    return PIFPAF_OK;
}

int pifpaf_cifdet_decode_device(pifpaf_cifdet_t* det, const float* field_dev, int32_t batch, int32_t h, int32_t w,
                                int32_t stride, const pifpaf_cifdet_params_t* params, void* stream_v) {
    PIFPAF_CHECK_ARG(det != nullptr, "cifdet handle is null");
    PIFPAF_CHECK_ARG(field_dev != nullptr && params != nullptr, "null argument");
    PIFPAF_CHECK_ARG(batch >= 1 && batch <= det->max_batch, "batch exceeds max_batch given at create()");
    PIFPAF_CHECK_ARG(h >= 1 && w >= 1 && h <= det->max_h && w <= det->max_w, "field shape exceeds max_h/max_w");
    PIFPAF_CHECK_ARG(stride >= 1 && stride <= det->max_stride, "stride exceeds max_stride");
    const pifpaf_cifdet_params_t& p = *params;
    PIFPAF_CHECK_ARG(p.occ_reduction >= 1.0 && p.cifhr_neighbors != 0, "bad occupancy reduction / neighbors");
    PIFPAF_CHECK_ARG(p.max_detections_before_nms >= 1 && p.max_detections_before_nms <= det->max_det,
                     "max_detections_before_nms exceeds the max_detections given at create()");
    PIFPAF_CUDA_TRY(cudaSetDevice(det->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    Dims d;
    d.B = batch; d.F = det->F; d.C = 0; d.K = det->F;
    d.h = h; d.w = w; d.hw = h * w; d.cif_stride = stride; d.caf_stride = stride;
    d.H = (h - 1) * stride + 1; d.W = (w - 1) * stride + 1;
    d.Wp = (d.W + TILE - 1) / TILE * TILE;
    d.Ho = (int)((double)d.H / p.occ_reduction) + 1; d.Wo = (int)((double)d.W / p.occ_reduction) + 1;
    d.tiles_x = d.Wp / TILE; d.tiles_y = (d.H + TILE - 1) / TILE;
    d.max_ann = det->max_det;
    det->last = d; det->has_last = true;
    if (det->epoch > 254) {                                    // one occupancy tag per decode
        PIFPAF_CUDA_TRY(cudaMemsetAsync(det->d_occ, 0, det->occ_bytes, st));
        det->epoch = 1;
    }
    const unsigned char tag = (unsigned char)det->epoch++;
    if (++det->hr_epoch == 0) {
        PIFPAF_CUDA_TRY(cudaMemsetAsync(det->d_tile_epoch, 0, sizeof(unsigned) * det->tile_epoch_elems, st));
        det->hr_epoch = 1;
    }
    GrowParams gp{};
    gp.occ_reduction = p.occ_reduction; gp.occ_min_scale_reduced = p.occ_min_scale / p.occ_reduction;
    // cifDetHr.accumulate(field, stride, 0.0, 1.0)   (src/cifdet.cpp:31)
    const float min_scale_f = (float)(0.0 / (double)stride);
    PIFPAF_CUDA_TRY(cudaMemsetAsync(det->d_work_count, 0, sizeof(int), st));
    k_cif_compact<<<dim3(d.F, d.B), NT, 0, st>>>(field_dev, d, 1, p.cifhr_threshold, (long long)p.cifhr_neighbors,
                                                 min_scale_f, 1.0, det->d_cells, det->d_boxes, det->d_cell_counts,
                                                 det->d_tile_epoch, det->hr_epoch, det->d_worklist, det->d_work_count);
    PIFPAF_LAUNCH_CHECK();
    k_cifhr_tiles<<<det->n_sm * 8, NT, 0, st>>>(d, p.cifhr_revision, det->d_cells, det->d_boxes, det->d_cell_counts,
                                                det->d_worklist, det->d_work_count, det->d_cifhr);
    PIFPAF_LAUNCH_CHECK();
    k_seed_candidates<<<dim3(d.F, d.B), NT, 0, st>>>(field_dev, d, det->d_cifhr, det->d_tile_epoch, det->hr_epoch,
                                                     p.cifhr_revision, p.seed_threshold, 0, 0, 1,
                                                     det->d_seg_v, det->d_seg_xys, det->d_seg_counts);
    PIFPAF_LAUNCH_CHECK();
    const size_t ss = sizeof(int) * (((size_t)d.F + 1 + 3) / 4 * 4 + 256 + 256 + 8) + 2 * 32 * 256 + 16;
    k_seed_sort<<<d.B, SORT_NT, ss, st>>>(d, det->d_seg_counts, det->d_seg_v, det->d_seg_xys, det->d_keys_a,
                                          det->d_vals_a, det->d_keys_b, det->d_vals_b, det->d_seed_f,
                                          det->d_seed_vxyw, det->d_seed_h, det->d_n_seeds);
    PIFPAF_LAUNCH_CHECK();
    const int max_det = (int)p.max_detections_before_nms;
    k_det_select<<<d.B, 32, 0, st>>>(d, gp, max_det, det->d_seed_f, det->d_seed_vxyw, det->d_seed_h, det->d_n_seeds,
                                     det->d_occ, tag, det->d_records, det->d_counts);
    PIFPAF_LAUNCH_CHECK();
    if (p.nms) {
        k_det_nms<<<d.B, DET_NMS_NT, det_nms_smem(max_det), st>>>(max_det, (float)p.iou_threshold, p.nms_by_category,
                                                                  (float)p.suppression, (float)p.instance_threshold,
                                                                  det->d_records, det->d_counts);
        PIFPAF_LAUNCH_CHECK();
    }
    det->last.max_ann = max_det;
    return PIFPAF_OK;
}

int pifpaf_cifdet_fetch(pifpaf_cifdet_t* det, int32_t* counts, float* records, int32_t cap, void* stream_v) {
    PIFPAF_CHECK_ARG(det != nullptr && det->has_last, "no decode to fetch");
    PIFPAF_CHECK_ARG(counts != nullptr, "counts is null");
    PIFPAF_CUDA_TRY(cudaSetDevice(det->device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    const int B = det->last.B, max_det = det->last.max_ann;
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(det->h_counts, det->d_counts, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(det->h_records, det->d_records, sizeof(float) * (size_t)B * max_det * DET_REC,
                                    cudaMemcpyDeviceToHost, st));
    PIFPAF_CUDA_TRY(cudaStreamSynchronize(st));
    bool overflow = false;
    for (int b = 0; b < B; b++) {
        counts[b] = det->h_counts[b];
        if (records == nullptr) continue;
        int n = det->h_counts[b];
        if (n > cap) { overflow = true; n = cap; }
        std::memcpy(records + (size_t)b * cap * DET_REC, det->h_records + (size_t)b * max_det * DET_REC,
                    sizeof(float) * (size_t)n * DET_REC);
    }
    if (overflow) { pifpaf::set_error("detection capacity exceeded (cap=%d)", cap); return PIFPAF_E_OVERFLOW; }
    return PIFPAF_OK;
}

int pifpaf_cifdet_call(pifpaf_cifdet_t* det, const float* field, int32_t stride, int32_t h, int32_t w,
                       const pifpaf_cifdet_params_t* params, float* records, int32_t cap, int32_t* n_out) {
    PIFPAF_CHECK_ARG(det != nullptr && field != nullptr && n_out != nullptr, "null argument");
    PIFPAF_CHECK_ARG(h >= 1 && w >= 1 && h <= det->max_h && w <= det->max_w, "field shape exceeds max_h/max_w");
    PIFPAF_CUDA_TRY(cudaSetDevice(det->device));
    cudaStream_t st = det->own_stream;
    PIFPAF_CUDA_TRY(cudaMemcpyAsync(det->d_in_field, field, sizeof(float) * (size_t)det->F * 6 * h * w,
                                    cudaMemcpyHostToDevice, st));
    int rc = pifpaf_cifdet_decode_device(det, det->d_in_field, 1, h, w, stride, params, st);
    if (rc != PIFPAF_OK) return rc;
    int32_t count = 0;
    rc = pifpaf_cifdet_fetch(det, &count, records, cap, st);
    *n_out = count;
    return rc;
}

}  // extern "C"
