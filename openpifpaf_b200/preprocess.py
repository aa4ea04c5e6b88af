"""GPU image preprocessing and batched annotation post-processing (SURVEY.md 8f rank 2).

Reference (paths relative to the reference's src/openpifpaf/):
  Predictor._preprocess_factory        predictor.py:85-102   NormalizeAnnotations, RescaleAbsolute, CenterPad /
                                                             CenterPadTight(16), EVAL_TRANSFORM
  transforms.RescaleAbsolute / _scale  transforms/scale.py:28-100,154-176   (fast=True, OpenCV absent:
                                                             PIL.Image.resize((w, h), BILINEAR), scale.py:56-59;
                                                             fast=True, OpenCV importable: cv2.resize(INTER_LINEAR),
                                                             scale.py:41-55;
                                                             fast=False: scipy.ndimage.zoom(order=1), scale.py:60-67)
  transforms.CenterPad / CenterPadTight  transforms/pad.py:15-110
  Annotation.inverse_transform / json_data / score / bbox   annotation.py:96-214

`GpuPreprocess` takes the RAW uint8 images of a batch, resizes them on the GPU bit-identically to Pillow
(pifpaf_image_resize_bilinear_u8; Pillow's ImagingResample restated, this module builds its coefficient tables) straight
into the centre of a padded uint8 canvas -- or, with fast_rescaling=False (RescaleAbsolute(fast=False),
transforms/scale.py:60-67), bit-identically to scipy.ndimage.zoom(order=1) (pifpaf_image_zoom_linear_u8, the whole
batch in one launch; `scipy_zoom_tables` / `zoom_linear_reference` restate scipy) -- or, with opencv=True,
bit-identically to cv2.resize(INTER_LINEAR) (pifpaf_image_resize_linear_cv_u8, one launch as well;
`opencv_linear_tables` / `opencv_linear_reference` restate OpenCV) -- and returns the canvas -- the input of
`CompiledNet.forward_uint8`, whose stem applies ToTensor + Normalize -- together with the per-image `meta` dicts the
reference's transforms would have produced.
`GpuJpegDecoder` decodes baseline JPEG files on the GPU bit-identically to PIL.Image.open(f).convert('RGB')
(datasets/image_list.py:18), the step before them; streams the GPU does not decode are decoded by Pillow.
`inverse_transform_batch` / `json_data_batch` are the array forms of `Annotation.inverse_transform` / `json_data` for all
annotations of an image at once (same float32 / float64 roundings as the reference under numpy 2).
"""
import ctypes
import io
import math
import numbers

import numpy as np
import torch

from . import _lib

PRECISION_BITS = 32 - 8 - 2          # Pillow src/libImaging/Resample.c
BILINEAR = 2                         # PIL.Image.Resampling.BILINEAR, RescaleAbsolute's default resample
TIGHT_PAD_FILL = (124, 116, 104)     # transforms/pad.py:100-101


def pil_bilinear_coeffs(in_size, out_size):
    """Pillow's precompute_coeffs(inSize, in0=0, in1=inSize, outSize, BILINEAR) followed by normalize_coeffs_8bpc
    (src/libImaging/Resample.c): bounds int32 [out, 2] (first input index, count) and fixed-point coefficients
    int32 [out, ksize].  IEEE double arithmetic in Pillow's order (the weight sum is accumulated left to right)."""
    in_size, out_size = int(in_size), int(out_size)
    scale = float(np.float32(in_size) - np.float32(0.0)) / out_size           # (double)(in1 - in0) / outSize, float box
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale                                               # bilinear support 1.0
    ksize = int(math.ceil(support)) * 2 + 1
    xx = np.arange(out_size, dtype=np.float64)
    center = 0.0 + (xx + 0.5) * scale
    ss = 1.0 / filterscale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)           # (int) truncates toward zero; clamped
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    k = np.zeros((out_size, ksize), dtype=np.float64)
    ww = np.zeros((out_size,), dtype=np.float64)
    for x in range(ksize):
        arg = ((x + xmin) - center + 0.5) * ss
        arg = np.where(arg < 0.0, -arg, arg)
        w = np.where(arg < 1.0, 1.0 - arg, 0.0)
        w = np.where(x < xmax, w, 0.0)
        k[:, x] = w
        ww = ww + w                                                           # sequential, like the C loop
    nz = ww != 0.0
    k[nz] = k[nz] / ww[nz, None]
    kk = np.where(k < 0, -0.5 + k * (1 << PRECISION_BITS), 0.5 + k * (1 << PRECISION_BITS)).astype(np.int64)
    kk = np.where(np.arange(ksize)[None, :] < xmax[:, None], kk, 0).astype(np.int32)
    bounds = np.stack([xmin, xmax], axis=1).astype(np.int32)
    return bounds, kk


def resize_bilinear_reference(image, target_w, target_h):
    """numpy restatement of Pillow's two-pass 8-bit resize with the tables above (used by the CPU parity test
    against PIL itself; the GPU kernels do the same integer arithmetic)."""
    img = np.asarray(image, dtype=np.uint8)
    h, w = img.shape[:2]

    def one_pass(a, bounds, kk, axis):
        a = np.moveaxis(a, axis, 0).astype(np.int64)
        out = np.empty((bounds.shape[0],) + a.shape[1:], dtype=np.uint8)
        for i in range(bounds.shape[0]):
            lo, n = int(bounds[i, 0]), int(bounds[i, 1])
            acc = (1 << (PRECISION_BITS - 1)) + np.tensordot(kk[i, :n].astype(np.int64), a[lo:lo + n], axes=(0, 0))
            out[i] = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
        return np.moveaxis(out, 0, axis)
    if target_w != w:
        img = one_pass(img, *pil_bilinear_coeffs(w, target_w), axis=1)
    if target_h != h:
        img = one_pass(img, *pil_bilinear_coeffs(h, target_h), axis=0)
    return img


ZOOM_TAP = np.dtype([('w0', '<f8'), ('w1', '<f8'), ('i0', '<i4'), ('i1', '<i4')])     # pifpaf_zoom_tap_t


def scipy_zoom_tables(n_in, n_out):
    """One axis of scipy.ndimage.zoom(..., order=1, mode='constant', cval=0, grid_mode=False) from n_in to n_out
    samples: per output index a pifpaf_zoom_tap_t (`ZOOM_TAP`) -- first input index i0, second index i1, weights
    w0 / w1, and i0 = -1 where scipy writes cval.  Established from scipy's wrapper (ndimage/_interpolation.py) and by
    probing its zoom_shift:
    - zoom = (n_in - 1) / (n_out - 1) in float64, and 1 where n_out - 1 == 0 (numpy.divide(..., where=zoom_div != 0)):
      a 1-sample output reads input 0, a 1-sample input is read at 0 by every output;
    - output index k samples the input at cc = k * zoom (grid_mode=False, no shift);
    - mode='constant': cc > n_in - 1 is outside the input, and the whole output row / column is cval.  The last
      index can land an ulp above n_in - 1 (28 -> 27 samples: 27 * (27 / 26) = 27.000000000000004), so some
      sizes get a black last row or column;
    - i0 = floor(cc), x = cc - i0, w0 = 1 - x and w1 = 1 - w0 (not x: the weights are completed to sum to 1).  At
      cc = n_in - 1, w1 = 0 and scipy reads a mirrored index; i1 is clamped to n_in - 1 here, which gives the same
      zero term."""
    n_in, n_out = int(n_in), int(n_out)
    if n_in < 1 or n_out < 1:
        raise RuntimeError(f'zoom from {n_in} to {n_out} samples: sizes must be at least 1')
    zoom = (n_in - 1) / (n_out - 1) if n_out != 1 else 1.0
    cc = np.arange(n_out, dtype=np.float64) * zoom
    outside = cc > n_in - 1
    i0 = np.floor(cc)
    w0 = 1.0 - (cc - i0)
    taps = np.zeros((n_out,), dtype=ZOOM_TAP)
    taps['w0'] = w0
    taps['w1'] = 1.0 - w0
    taps['i0'] = np.where(outside, -1, i0)
    taps['i1'] = np.where(outside, -1, np.minimum(i0 + 1, n_in - 1))
    return taps


def zoom_linear_reference(image, target_w, target_h):
    """numpy restatement of scipy.ndimage.zoom(image, (target_h / h, target_w / w, 1), order=1) on a uint8 [h, w, 3]
    image (transforms/scale.py:60-67), from `scipy_zoom_tables`; the GPU kernel k_zoom_linear does the same.
    - The channel axis zooms 3 -> 3 by exactly 1: its weights are exactly 1 and 0, so each of the four (y, x) terms
      is (v * wy) * wx (scipy multiplies the weights onto the value axis by axis), and its zero-weight terms add
      +0.0.  The terms are summed from 0.0 in scipy's filter order: (y0, x0), (y0, x1), (y1, x0), (y1, x1).
    - A sample with a row or column outside the input is cval = 0.
    - uint8 conversion: t > 0 ? t + 0.5 : 0, clamped to 255, truncated -- ties round up, unlike numpy.round, and
      the float64 sum decides which side of a .5 a sample lands on.
    - scipy returns the input unchanged when both factors are 1; the tables then give exactly that."""
    img = np.asarray(image, dtype=np.uint8)
    h, w = img.shape[:2]
    ty, tx = scipy_zoom_tables(h, target_h), scipy_zoom_tables(w, target_w)
    v = img.astype(np.float64)
    wy0, wy1 = ty['w0'][:, None, None], ty['w1'][:, None, None]
    wx0, wx1 = tx['w0'][None, :, None], tx['w1'][None, :, None]
    y0, y1 = np.maximum(ty['i0'], 0), np.maximum(ty['i1'], 0)
    x0, x1 = np.maximum(tx['i0'], 0), np.maximum(tx['i1'], 0)
    t = 0.0 + (v[y0][:, x0] * wy0) * wx0
    t = t + (v[y0][:, x1] * wy0) * wx1
    t = t + (v[y1][:, x0] * wy1) * wx0
    t = t + (v[y1][:, x1] * wy1) * wx1
    t = np.where((ty['i0'] < 0)[:, None, None] | (tx['i0'] < 0)[None, :, None], 0.0, t)
    t = np.minimum(np.where(t > 0, t + 0.5, 0.0), 255.0)
    return t.astype(np.uint8)


CV_TAP = np.dtype([('i0', '<i4'), ('i1', '<i4'), ('c0', '<i2'), ('c1', '<i2')])     # pifpaf_cv_tap_t
CV_COEF_ONE = 1 << 11                # INTER_RESIZE_COEF_SCALE, modules/imgproc/src/resize.cpp


def opencv_linear_tables(n_in, n_out, horizontal=True):
    """One axis of cv2.resize(..., interpolation=INTER_LINEAR) on uint8 from n_in to n_out samples
    (modules/imgproc/src/resize.cpp: cv::resize -> resizeGeneric_ with HResizeLinear / VResizeLinear): per output
    index a pifpaf_cv_tap_t (`CV_TAP`) -- the two source indices i0 / i1 and their 11-bit coefficients c0 / c1.
    - scale = 1 / (n_out / n_in) in double; f = (float)((k + 0.5) * scale - 0.5); s = floor(f); f -= s in float.
    - c0 = saturate_cast<short>((1.f - f) * 2048), c1 = saturate_cast<short>(f * 2048): float products rounded to
      nearest, ties to even.
    - Border clamp, columns (horizontal=True): where s < 0 or s >= n_in - 1 OpenCV sets f = 0 and s to the border
      column, so the tap is (border, 2048) and (border, 0).
    - Rows (horizontal=False) keep f: s and s + 1 are clipped into [0, n_in - 1] and both coefficients stay, so a
      border row of an upscale reads the edge row twice with fractional weights.  The vertical pass truncates each
      product on its own (`opencv_linear_reference`), so this is not the same as weights (2048, 0): it is the border
      rule that makes the first and last rows of upscales differ by 1 from a clamped restatement.
    c0 + c1 = 2048 in every tap."""
    n_in, n_out = int(n_in), int(n_out)
    if n_in < 1 or n_out < 1:
        raise RuntimeError(f'resize from {n_in} to {n_out} samples: sizes must be at least 1')
    scale = 1.0 / (n_out / n_in)
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    f = f - s
    s = s.astype(np.int64)
    if horizontal:
        border = (s < 0) | (s >= n_in - 1)
        f = np.where(border, np.float32(0), f)
        s = np.clip(s, 0, n_in - 1)
    one = np.float32(CV_COEF_ONE)
    taps = np.zeros((n_out,), dtype=CV_TAP)
    taps['i0'] = np.clip(s, 0, n_in - 1)
    taps['i1'] = np.clip(s + 1, 0, n_in - 1)
    taps['c0'] = np.clip(np.rint((np.float32(1) - f) * one), -32768, 32767)
    taps['c1'] = np.clip(np.rint(f * one), -32768, 32767)
    return taps


def opencv_linear_reference(image, target_w, target_h):
    """numpy restatement of cv2.resize(image, (target_w, target_h), interpolation=cv2.INTER_LINEAR) on a uint8
    [h, w, 3] image (transforms/scale.py:41-55, RescaleAbsolute(fast=True) when OpenCV is importable), from
    `opencv_linear_tables`; the GPU kernel k_resize_linear_cv does the same integer arithmetic.
    - Horizontal pass, exact in int32: H = v[i0] * c0 + v[i1] * c1 per source row and channel.
    - Vertical pass, as OpenCV's SIMD VResizeLinearVec_32s8u computes it on every element (also the last ones of a
      row, and 1-pixel images): each row's H is shifted right by 4 into int16, multiplied by its coefficient keeping
      the high 16 bits, the two products added, then (t + 2) >> 2 saturated to uint8.  Not the textbook rounding
      (H0 * c0 + H1 * c1 + 2^21) >> 22: each product is truncated on its own.
    - Exactly 2x down on both axes OpenCV switches INTER_LINEAR to INTER_AREA's fast path, (a + b + c + d + 2) >> 2.
      The linear taps are then (i, 1024) and (i + 1, 1024) on both axes and the vertical pass gives the same sum, so
      no pixel changes and no separate rule is needed.
    - An unchanged size is a copy; the taps are then (k, 2048) and give exactly that."""
    img = np.asarray(image, dtype=np.uint8)
    h, w = img.shape[:2]
    tx, ty = opencv_linear_tables(w, target_w, True), opencv_linear_tables(h, target_h, False)
    v = img.astype(np.int64)
    hp = v[:, tx['i0']] * tx['c0'][None, :, None] + v[:, tx['i1']] * tx['c1'][None, :, None]
    c0y, c1y = ty['c0'][:, None, None], ty['c1'][:, None, None]
    t = (((hp[ty['i0']] >> 4) * c0y) >> 16) + (((hp[ty['i1']] >> 4) * c1y) >> 16)
    return np.clip((t + 2) >> 2, 0, 255).astype(np.uint8)


def rescale_target(w, h, long_edge):
    """RescaleAbsolute.__call__ (transforms/scale.py:163-176)"""
    s = long_edge / max(h, w)
    if h > w:
        return int(w * s), int(long_edge)
    return int(long_edge), int(h * s)


def center_pad_ltrb(w, h, target_w, target_h):
    """CenterPad.center_pad / CenterPadTight.center_pad (transforms/pad.py:37-49,87-99)"""
    left = max(0, int((target_w - w) / 2.0))
    top = max(0, int((target_h - h) / 2.0))
    right = max(0, target_w - w - left)
    bottom = max(0, target_h - h - top)
    return left, top, right, bottom


def reference_meta(w, h, target_w, target_h, ltrb, rescaled=True):
    """The meta dict after NormalizeAnnotations -> _scale -> CenterPad (transforms/annotations.py:52-77,
    transforms/scale.py:73-96, transforms/pad.py:26-33), float64 numpy like the reference.
    rescaled: RescaleAbsolute is part of the pipeline (a long edge is set).  Its _scale runs even when the size does not
    change, and divides by zero on a 1-pixel-wide or -high image like the reference; without it no factor applies."""
    meta = {'offset': np.array((0.0, 0.0)), 'scale': np.array((1.0, 1.0)),
            'rotation': {'angle': 0.0, 'width': None, 'height': None},
            'valid_area': np.array((0.0, 0.0, w - 1, h - 1)), 'hflip': False, 'width_height': np.array((w, h))}
    if rescaled:
        x_scale = (target_w - 1) / (w - 1)
        y_scale = (target_h - 1) / (h - 1)
        sf = np.array((x_scale, y_scale))
        meta['offset'] *= sf
        meta['scale'] *= sf
        meta['valid_area'][:2] *= sf
        meta['valid_area'][2:] *= sf
    meta['offset'] -= ltrb[:2]
    meta['valid_area'][:2] += ltrb[:2]
    return meta


def pad_fills(fill, n_images, batched):
    """The `fill` argument of GpuPreprocess -> one (r, g, b) per image.  An int (grey) or a tuple (r, g, b) is one
    colour for every image; a list holds one int or (r, g, b) per image and has exactly n_images entries.  None draws
    like the reference: CenterPad a random grey per image with torch.randint(0, 255) (transforms/pad.py:52),
    CenterPadTight (124, 116, 104) (pad.py:100-101)."""
    if fill is None:
        fill = [int(torch.randint(0, 255, (1,)).item()) if batched else TIGHT_PAD_FILL for _ in range(n_images)]
    elif isinstance(fill, list):
        if len(fill) != n_images:
            raise RuntimeError(f'fill has {len(fill)} colours for {n_images} images')
    else:
        fill = [fill] * n_images
    out = []
    for f in fill:
        c = (int(f),) * 3 if isinstance(f, numbers.Integral) else tuple(int(v) for v in f)
        if len(c) != 3:
            raise RuntimeError(f'a pad colour is an int or an (r, g, b) triple, not {f!r}')
        out.append(c)
    return out


def resize_path(w, h, target_w, target_h, dst_pitch_bytes):
    """The launch sequence pifpaf_image_resize_bilinear_u8 takes for a [h, w] image resized to [target_h, target_w]
    into a destination with the given row pitch: 'hv' (horizontal pass into tmp, vertical pass into the destination),
    'h_dense' (horizontal pass straight into a dense destination), 'h_pitched' (horizontal pass into tmp, then a row
    copy), 'v' (vertical pass from the source) or 'copy'."""
    need_h, need_v = target_w != w, target_h != h
    if need_h and need_v:
        return 'hv'
    if need_h:
        return 'h_dense' if dst_pitch_bytes == target_w * 3 else 'h_pitched'
    return 'v' if need_v else 'copy'


class GpuPreprocess:
    """:param long_edge: RescaleAbsolute target (None: no rescale, like --long-edge unset)
    :param batched: True -> CenterPad(long_edge) squares (predictor.py:91-93, batch size > 1);
                    False -> CenterPadTight(16) (predictor.py:94-95)
    :param fast_rescaling: the reference's Predictor.fast_rescaling / RescaleAbsolute(fast=...): True resizes like
                    PIL.Image.resize (pifpaf_image_resize_bilinear_u8); False like scipy.ndimage.zoom(order=1), the
                    precise rescale of --precise-rescaling and of every evaluation preprocess
                    (pifpaf_image_zoom_linear_u8, the whole batch in one launch)
    :param opencv: with fast_rescaling, resize like cv2.resize(INTER_LINEAR) instead of Pillow -- what
                    RescaleAbsolute(fast=True) does when OpenCV is importable (pifpaf_image_resize_linear_cv_u8, the
                    whole batch in one launch).  Without fast_rescaling scipy is used either way, as in the reference
    :param resample: RescaleAbsolute's resample; only BILINEAR (2, its default) is built"""

    def __init__(self, long_edge=None, batched=True, *, fast_rescaling=True, opencv=False, resample=BILINEAR, device=0,
                 multiple=16):
        if batched and not long_edge:
            raise RuntimeError('--long-edge must be provided for batch size > 1')      # predictor.py:92
        if resample != BILINEAR:
            raise RuntimeError(f'resample={resample!r} is not built: only BILINEAR ({BILINEAR}; scipy order 1) is')
        self.long_edge = int(long_edge) if long_edge else None
        self.batched = bool(batched)
        self.fast_rescaling = bool(fast_rescaling)
        self.opencv = bool(opencv) and self.fast_rescaling
        self.multiple = int(multiple)
        self.device = torch.device('cuda', device)
        self._coeff_cache = {}
        self._tap_cache = {}

    def _taps(self, n_in, n_out, horizontal):
        """one axis's taps for the one-launch paths: scipy's (the same for both axes) or OpenCV's"""
        key = (n_in, n_out, horizontal and self.opencv)
        if key not in self._tap_cache:
            self._tap_cache[key] = (opencv_linear_tables(n_in, n_out, horizontal) if self.opencv
                                    else scipy_zoom_tables(n_in, n_out))
        return self._tap_cache[key]

    def _coeffs(self, n_in, n_out):
        key = (n_in, n_out)
        if key not in self._coeff_cache:
            b, k = pil_bilinear_coeffs(n_in, n_out)
            self._coeff_cache[key] = (torch.from_numpy(b).to(self.device), torch.from_numpy(k).to(self.device), k.shape[1])
        return self._coeff_cache[key]

    def plan(self, sizes):
        """sizes: [(w, h)] of the raw images -> per-image (target_w, target_h, ltrb) and the canvas (W, H)"""
        out = []
        for (w, h) in sizes:
            tw, th = rescale_target(w, h, self.long_edge) if self.long_edge else (w, h)
            if self.batched:
                cw = ch = self.long_edge
            else:
                cw = math.ceil((tw - 1) / self.multiple) * self.multiple + 1
                ch = math.ceil((th - 1) / self.multiple) * self.multiple + 1
            out.append((tw, th, center_pad_ltrb(tw, th, cw, ch), (cw, ch)))
        canvases = {o[3] for o in out}
        if len(canvases) != 1:
            raise RuntimeError('images of one batch must share the padded size (use batched=True with a long edge)')
        return out, canvases.pop()

    def __call__(self, images, fill=None, stream=None):
        """images: list of uint8 [h, w, 3] arrays / tensors (host or CUDA).  fill: pad colour -- an int (grey) or an
        (r, g, b) tuple for every image, or a list of those per image (`pad_fills`; default like the reference).
        Returns (canvas uint8 CUDA [B, H, W, 3], metas)."""
        imgs = [torch.as_tensor(np.ascontiguousarray(im)) if not isinstance(im, torch.Tensor) else im.contiguous()
                for im in images]
        for im in imgs:
            if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
                raise RuntimeError('images must be uint8 [h, w, 3]')
        sizes = [(int(im.shape[1]), int(im.shape[0])) for im in imgs]
        plans, (cw, ch) = self.plan(sizes)
        B = len(imgs)
        fill = pad_fills(fill, B, self.batched)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        if any(im.is_cuda for im in imgs):
            st.wait_stream(torch.cuda.current_stream(self.device))     # CUDA inputs (and .contiguous()) are written there
        if self.opencv or not self.fast_rescaling:
            return self._one_launch(imgs, sizes, plans, (cw, ch), fill, st)
        L = _lib.lib()
        sp = ctypes.c_void_p(st.cuda_stream)
        with torch.cuda.stream(st):
            canvas = torch.empty((B, ch, cw, 3), dtype=torch.uint8, device=self.device)
            metas, keep = [], []
            for b, (im, (w, h), (tw, th, ltrb, _)) in enumerate(zip(imgs, sizes, plans)):
                _lib.check(L.pifpaf_image_fill_rgb(canvas[b].data_ptr(), ch * cw, fill[b][0], fill[b][1], fill[b][2], sp))
                src = im.pin_memory().to(self.device, non_blocking=True) if not im.is_cuda else im
                xb = xk = yb = yk = None
                xks = yks = 0
                if tw != w:
                    xb, xk, xks = self._coeffs(w, tw)
                if th != h:
                    yb, yk, yks = self._coeffs(h, th)
                tmp = torch.empty((h * tw * 3,), dtype=torch.uint8, device=self.device)
                dst = canvas[b].data_ptr() + (ltrb[1] * cw + ltrb[0]) * 3
                _lib.check(L.pifpaf_image_resize_bilinear_u8(
                    src.data_ptr(), h, w, dst, cw * 3, th, tw,
                    xb.data_ptr() if xb is not None else None, xk.data_ptr() if xk is not None else None, xks,
                    yb.data_ptr() if yb is not None else None, yk.data_ptr() if yk is not None else None, yks,
                    tmp.data_ptr(), sp))
                keep.append((src, tmp))
                metas.append(reference_meta(w, h, tw, th, np.asarray(ltrb), rescaled=self.long_edge is not None))
            self._keepalive = keep
        return canvas, metas

    def _one_launch(self, imgs, sizes, plans, canvas_size, fill, st):
        """the scipy (fast_rescaling=False) and OpenCV paths of __call__: every image's taps (one table per distinct
        (in, out) pair and, for OpenCV, axis) and descriptor staged, and the whole canvas written, by one
        pifpaf_image_zoom_linear_u8 / pifpaf_image_resize_linear_cv_u8"""
        cw, ch = canvas_size
        B = len(imgs)
        tables, offsets, n_taps = [], {}, 0

        def tap_offset(n_in, n_out, horizontal):
            nonlocal n_taps
            key = (n_in, n_out, horizontal and self.opencv)
            if key not in offsets:
                offsets[key] = n_taps
                tables.append(self._taps(n_in, n_out, horizontal))
                n_taps += n_out
            return offsets[key]

        L = _lib.lib()
        descs = ((_lib.CvImage if self.opencv else _lib.ZoomImage) * B)()
        metas, srcs = [], []
        with torch.cuda.stream(st):
            canvas = torch.empty((B, ch, cw, 3), dtype=torch.uint8, device=self.device)
            for d, im, (w, h), (tw, th, ltrb, _), f in zip(descs, imgs, sizes, plans, fill):
                src = im.pin_memory().to(self.device, non_blocking=True) if not im.is_cuda else im
                srcs.append(src)
                d.src, d.h, d.w, d.th, d.tw, d.left, d.top = src.data_ptr(), h, w, th, tw, ltrb[0], ltrb[1]
                d.ytab, d.xtab = tap_offset(h, th, False), tap_offset(w, tw, True)
                if self.opencv:
                    d.pitch = w * 3
                if not all(0 <= c <= 255 for c in f):
                    raise RuntimeError(f'fill colour out of range: {f}')
                d.fill[:3] = f
                metas.append(reference_meta(w, h, tw, th, np.asarray(ltrb), rescaled=self.long_edge is not None))
            taps = np.ascontiguousarray(np.concatenate(tables))
            ws_bytes = ctypes.sizeof(descs) + taps.nbytes
            workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=self.device)
            entry = L.pifpaf_image_resize_linear_cv_u8 if self.opencv else L.pifpaf_image_zoom_linear_u8
            _lib.check(entry(descs, B, taps.ctypes.data, taps.size, workspace.data_ptr(), ws_bytes, canvas.data_ptr(),
                             ch, cw, ctypes.c_void_p(st.cuda_stream)))
            self._keepalive = (srcs, workspace)
        return canvas, metas


# ----------------------------------------------------------------------------------------------------- JPEG decode
def read_stream(f):
    """a path or a bytes-like JPEG stream -> bytes"""
    if isinstance(f, (bytes, bytearray, memoryview)):
        return bytes(f)
    with open(f, 'rb') as fh:
        return fh.read()


def pillow_rgb(data):
    """the reference's decode (datasets/image_list.py:18): uint8 [h, w, 3]"""
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        return np.asarray(im.convert('RGB'))


def jpeg_footprint(data):
    """(w * h, 8x8 blocks of the MCU grid) of a JPEG stream as pifpaf_jpeg_decode lays it out, from its frame header
    (Pillow's parse; (0, 0) if Pillow cannot open it -- the decoder then reports why).  Sizes `GpuJpegDecoder` for a
    batch exactly."""
    from PIL import Image
    try:
        with Image.open(io.BytesIO(data)) as im:
            w, h = im.size
            layer = list(getattr(im, 'layer', None) or [])          # (id, h sampling, v sampling, table) per component
    except Exception:                                                  # not an image Pillow can open
        return 0, 0
    if len(layer) <= 1:                                                # one component: one block per MCU
        return w * h, -(-w // 8) * -(-h // 8)
    hmax, vmax = max(c[1] for c in layer), max(c[2] for c in layer)
    mcus = -(-w // (8 * hmax)) * -(-h // (8 * vmax))
    return w * h, mcus * sum(c[1] * c[2] for c in layer)


class GpuJpegDecoder:
    """Decode JPEG files or byte strings on the GPU (pifpaf_jpeg_decode), bit-identically to
    PIL.Image.open(f).convert('RGB').  Baseline / extended-sequential Huffman streams with 8-bit samples in one scan,
    grayscale or YCbCr 4:4:4 / 4:2:2 / 4:2:0, take the 'gpu' route; every other stream (progressive, arithmetic,
    CMYK, Adobe RGB, 4:4:0, ...) the 'pillow' route, decoded by Pillow on the host like the reference.

    :param max_images: images per call
    :param max_bytes: entropy-coded bytes per call (the scans of all streams of a call)
    :param max_pixels: w * h of the largest image
    :param max_blocks: 8x8 blocks per call, summed over its images (`jpeg_footprint`); default: max_images images of
                       max_pixels pixels on a square MCU grid at 4:4:4
    :param out_pixels: pixels per call, summed over its images (the output buffer); default max_images * max_pixels
    The returned GPU-route images are views of one output buffer, valid until the next call."""

    def __init__(self, max_images, max_bytes, max_pixels, *, max_blocks=None, out_pixels=None, device=0):
        self.device = torch.device('cuda', device)
        self.max_images, self.max_bytes, self.max_pixels = int(max_images), int(max_bytes), int(max_pixels)
        if max_blocks is None:
            side = -(-math.isqrt(self.max_pixels - 1) // 8) + 1 if self.max_pixels > 1 else 1
            max_blocks = self.max_images * 3 * side * side
        self.max_blocks = int(max_blocks)
        self.out_pixels = int(out_pixels) if out_pixels is not None else self.max_images * self.max_pixels
        self._handle = ctypes.c_void_p()
        _lib.check(_lib.lib().pifpaf_jpeg_create(ctypes.byref(self._handle), device, self.max_images,
                                                 self.max_bytes, self.max_pixels, self.max_blocks))
        self._out = torch.empty((self.out_pixels * 3,), dtype=torch.uint8, device=self.device)
        self.last_routes = []

    def fits(self, n_images, n_bytes, max_pixels, n_blocks, n_pixels):
        """can one call take n_images streams of n_bytes in all, the largest of max_pixels, n_blocks and n_pixels
        summed (`jpeg_footprint`)"""
        return (n_images <= self.max_images and n_bytes <= self.max_bytes and max_pixels <= self.max_pixels
                and n_blocks <= self.max_blocks and n_pixels <= self.out_pixels)

    def __call__(self, files_or_bytes, *, max_rounds=-1, stream=None, host_pillow=False):
        """-> (images, routes): per stream a uint8 [h, w, 3] image (CUDA; with host_pillow the Pillow-route images
        stay host numpy arrays) and 'gpu' or 'pillow'.  The GPU decode is enqueued on `stream` (default: the current
        stream).  max_rounds caps the self-synchronising Huffman decode (-1: default, 0: serial); the images do not
        depend on it.  A malformed stream raises RuntimeError before anything is enqueued."""
        datas = [read_stream(f) for f in files_or_bytes]
        n = len(datas)
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        ptrs = (ctypes.c_void_p * max(n, 1))(*[ctypes.cast(ctypes.c_char_p(d), ctypes.c_void_p) for d in datas])
        sizes = (ctypes.c_int64 * max(n, 1))(*[len(d) for d in datas])
        routes = (ctypes.c_int32 * max(n, 1))()
        hw = (ctypes.c_int32 * max(2 * n, 1))()
        offs = (ctypes.c_int64 * max(n, 1))()
        _lib.check(_lib.lib().pifpaf_jpeg_decode(self._handle, n, ptrs, sizes, self._out.data_ptr(), self._out.numel(),
                                                 int(max_rounds), routes, hw, offs, ctypes.c_void_p(st.cuda_stream)))
        images, names = [], []
        for i in range(n):
            if routes[i] == 0:
                h, w, o = hw[2 * i], hw[2 * i + 1], offs[i]
                images.append(self._out[o:o + h * w * 3].view(h, w, 3))
                names.append('gpu')
            else:
                img = pillow_rgb(datas[i])
                if not host_pillow:
                    with torch.cuda.stream(st):
                        img = torch.from_numpy(np.ascontiguousarray(img)).to(self.device)
                images.append(img)
                names.append('pillow')
        self.last_routes = names
        return images, names

    def stats(self):
        """counters of the last call (synchronises): images per route, subsequences, self-synchronisation rounds that
        decoded something, serial fallback decodes"""
        s = (ctypes.c_int64 * 5)()
        _lib.check(_lib.lib().pifpaf_jpeg_last_stats(self._handle, s, 5))
        return dict(gpu=s[0], pillow=s[1], subsequences=s[2], sync_rounds=s[3], fallbacks=s[4])

    def close(self):
        if self._handle:
            _lib.lib().pifpaf_jpeg_destroy(self._handle)
            self._handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:                   # interpreter shutdown
            pass


# ----------------------------------------------------------------------------- annotations, all of an image at once

def inverse_transform_batch(ann, meta):
    """Annotation.inverse_transform (annotation.py:162-214; no rotation) for the packed decoder output of one image.
    ann: [N, K, 4] float32 (v, x, y, s) as the decoder returns it.  Returns (data [N, K, 3] float32 (x, y, v),
    joint_scales [N, K] float32) in original-image coordinates.  Rounding like the reference under numpy 2: the
    float32 arrays meet float64 meta scalars, each statement computes in float64 and stores float32."""
    ann = np.asarray(ann, dtype=np.float32)
    data = np.empty(ann.shape[:2] + (3,), dtype=np.float32)
    data[..., 0] = ann[..., 1]
    data[..., 1] = ann[..., 2]
    data[..., 2] = ann[..., 0]
    scales = ann[..., 3].copy()
    if meta['rotation']['angle'] != 0.0:
        raise RuntimeError('rotated inputs are not part of the inference path')
    ox, oy = np.float64(meta['offset'][0]), np.float64(meta['offset'][1])
    sx, sy = np.float64(meta['scale'][0]), np.float64(meta['scale'][1])
    data[..., 0] = data[..., 0].astype(np.float64) + ox
    data[..., 1] = data[..., 1].astype(np.float64) + oy
    data[..., 0] = data[..., 0].astype(np.float64) / sx
    data[..., 1] = data[..., 1].astype(np.float64) / sy
    scales = (scales.astype(np.float64) / sx).astype(np.float32)
    if meta['hflip']:
        w = meta['width_height'][0]
        data[..., 0] = -data[..., 0] + (w - 1)
        if meta.get('horizontal_swap'):
            for i in range(data.shape[0]):
                data[i] = meta['horizontal_swap'](data[i])
    return data, scales


def json_data_batch(data, joint_scales, score_weights=None, category_id=1, coordinate_digits=2):
    """Annotation.json_data (annotation.py:121-143) with score (annotation.py:96-111) and bbox_from_keypoints
    (annotation.py:150-160) for all annotations of an image; returns a list of dicts equal to the reference's."""
    data = np.asarray(data, dtype=np.float32)
    n, K = data.shape[:2]
    sw = np.ones((K,)) if score_weights is None else np.asarray(score_weights, dtype=np.float64).copy()
    sw = sw / np.sum(sw)
    out = []
    v_mask = data[..., 2] > 0.0
    kp = data.copy()
    kp[..., 2] = np.where(v_mask, np.maximum(np.float32(0.01), kp[..., 2]), kp[..., 2])
    kp = np.around(kp.astype(np.float64), coordinate_digits)
    js = np.asarray(joint_scales, dtype=np.float32)
    for i in range(n):
        m = data[i, :, 2] > 0
        if not np.any(m):
            bbox = [0, 0, 0, 0]
        else:
            x = np.min(data[i, :, 0][m] - js[i][m])
            y = np.min(data[i, :, 1][m] - js[i][m])
            bbox = [x, y, np.max(data[i, :, 0][m] + js[i][m]) - x, np.max(data[i, :, 1][m] + js[i][m]) - y]
        score = np.sum(sw * np.sort(data[i, :, 2])[::-1])
        out.append({'keypoints': kp[i].reshape(-1).tolist(),
                    'bbox': [round(float(c), coordinate_digits) for c in bbox],
                    'score': max(0.001, round(score, 3)),
                    'category_id': category_id})
    return out
