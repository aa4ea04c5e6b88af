"""CPU: the reference's fast rescale where OpenCV is importable (transforms.RescaleAbsolute(fast=True) ->
cv2.resize(INTER_LINEAR), transforms/scale.py:41-55) restated by `preprocess.opencv_linear_tables` /
`opencv_linear_reference`: against cv2 itself on a seeded size sweep that must contain a clamped border row and an
exact 2x reduction (OpenCV's INTER_AREA fast path), against tests/golden/opencv_resize.npz where OpenCV is missing,
and against the reference's own transforms with its module-level cv2 in place."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from openpifpaf_b200 import _lib
from openpifpaf_b200 import preprocess as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'opencv_resize.npz')

# (w, h) of common photos, rescaled as RescaleAbsolute would for the long edges below
PHOTO_SIZES = [(640, 480), (480, 640), (640, 427), (427, 640), (500, 375), (375, 500), (612, 612), (800, 600),
               (1024, 768), (1280, 720), (1920, 1080), (4032, 3024), (3024, 4032), (640, 360), (333, 500), (28, 27)]
LONG_EDGES = (321, 641, 801)


def sweep_sizes(n=260, seed=0):
    """(h, w, target_w, target_h): n random sizes in 1..900 (up, down and mixed), exact 2x reductions on both axes
    and on one, 1-pixel rows, columns, inputs and outputs, 4032 x 3024 photos, and every RescaleAbsolute target of
    PHOTO_SIZES at LONG_EDGES"""
    rng = np.random.default_rng(seed)
    out = [tuple(int(v) for v in rng.integers(1, 901, 4)) for _ in range(n)]
    for th, tw in rng.integers(1, 451, (6, 2)):
        th, tw = int(th), int(tw)
        out += [(2 * th, 2 * tw, tw, th), (2 * th, tw + 7, tw, th), (th + 3, 2 * tw, tw, th)]
    out += [(1, int(w), int(tw), 1) for w, tw in rng.integers(1, 901, (3, 2))]           # 1 x N -> 1 x M
    out += [(int(h), 1, 1, int(th)) for h, th in rng.integers(1, 901, (3, 2))]           # N x 1 -> M x 1
    out += [(1, 1, 1, 1), (1, 1, 13, 11), (1, 37, 5, 1), (29, 1, 1, 7), (40, 30, 1, 1), (1, 900, 1, 900),
            (900, 1, 900, 1), (2, 2, 1, 1), (2, 2, 900, 3), (900, 900, 1, 2), (480, 640, 641, 481),
            (3024, 4032, 641, 481), (4032, 3024, 481, 641), (962, 1282, 641, 481)]
    for le in LONG_EDGES:
        out += [(h, w) + pp.rescale_target(w, h, le) for (w, h) in PHOTO_SIZES]
    return out


def cv2_resize(img, tw, th):
    import cv2
    return cv2.resize(img, (tw, th), interpolation=cv2.INTER_LINEAR)


def clamped_border_rows(h, th):
    """output rows that read one source row twice with fractional weights (upscale borders)"""
    t = pp.opencv_linear_tables(h, th, horizontal=False)
    return (t['i0'] == t['i1']) & (t['c1'] > 0)


def test_opencv_restatement_equals_cv2_on_a_sweep():
    cv2 = pytest.importorskip('cv2')
    print('cv2', cv2.__version__)
    rng = np.random.default_rng(29)
    sizes = sweep_sizes()
    assert len(sizes) >= 300
    bad, border, area_fast = [], 0, 0
    for (h, w, tw, th) in sizes:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        want = cv2_resize(img, tw, th)
        got = pp.opencv_linear_reference(img, tw, th)
        if got.shape != want.shape or not np.array_equal(got, want):
            bad.append((h, w, tw, th))
        border += int(clamped_border_rows(h, th).any())
        area_fast += int(h == 2 * th and w == 2 * tw)
    assert not bad, f'{len(bad)} sizes differ from cv2, first: {bad[:5]}'
    print(f'{len(sizes)} sizes, {border} with a clamped border row, {area_fast} exact 2x reductions')
    assert border >= 1 and area_fast >= 1


def test_clamped_border_row_is_not_a_clamped_coordinate():
    """the first and last rows of an upscale: clamping the row coordinate like the columns (weights 2048 and 0)
    differs from cv2 -- the rule opencv_linear_tables states for rows"""
    cv2 = pytest.importorskip('cv2')
    img = np.random.default_rng(4).integers(0, 256, (480, 640, 3), dtype=np.uint8)
    want = cv2_resize(img, 641, 481)
    rows = clamped_border_rows(480, 481)
    assert rows[0] and rows[-1] and not rows[1:-1].any()
    x = pp.opencv_linear_tables(640, 641, horizontal=True)
    v = img.astype(np.int64)
    hp = v[:, x['i0']] * x['c0'][None, :, None] + v[:, x['i1']] * x['c1'][None, :, None]
    clamped = np.clip(((((hp[[0, -1]] >> 4) * 2048) >> 16) + 2) >> 2, 0, 255)
    assert (clamped != want[[0, -1]]).any()
    assert np.array_equal(pp.opencv_linear_reference(img, 641, 481), want)


def test_opencv_restatement_equals_stored_cv2_outputs():
    """tests/golden/opencv_resize.npz (tools/make_opencv_resize_golden.py): cv2's outputs on seeded inputs"""
    z = np.load(GOLDEN)
    print('stored from cv2', z['cv2_version'], '|', z['cv2_ipp'])
    shapes = z['shapes']
    assert len(shapes) >= 15
    for i, (seed, (h, w, th, tw)) in enumerate(zip(z['seeds'], shapes)):
        img = np.random.default_rng(int(seed)).integers(0, 256, (h, w, 3), dtype=np.uint8)
        np.testing.assert_array_equal(pp.opencv_linear_reference(img, int(tw), int(th)), z[f'out_{i}'],
                                      err_msg=f'case {i} {(h, w, th, tw)}')
    assert any(clamped_border_rows(h, th).any() for (h, w, th, tw) in shapes)
    assert any(h == 2 * th and w == 2 * tw for (h, w, th, tw) in shapes)


def test_opencv_tables():
    for n_in, n_out in ((1, 1), (1, 9), (9, 1), (2, 1), (480, 481), (641, 37), (4032, 641), (64, 32), (7, 900)):
        for horizontal in (True, False):
            t = pp.opencv_linear_tables(n_in, n_out, horizontal)
            assert t.dtype.itemsize == 12 and t.shape == (n_out,)
            assert ((t['c0'].astype(int) + t['c1']) == 2048).all() and (t['c0'] >= 0).all() and (t['c1'] >= 0).all()
            assert (t['i0'] >= 0).all() and (t['i1'] < n_in).all() and (t['i1'] >= t['i0']).all()
            if horizontal:                           # clamped columns read the border column with weight 2048
                border = t['i0'] == t['i1']
                assert (t['c0'][border] == 2048).all()
    t = pp.opencv_linear_tables(50, 50, False)       # unchanged: the identity
    assert np.array_equal(t['i0'], np.arange(50)) and (t['c0'] == 2048).all()
    t = pp.opencv_linear_tables(64, 32, False)       # exactly 2x: (2k, 1024) and (2k + 1, 1024)
    assert np.array_equal(t['i0'], 2 * np.arange(32)) and (t['c0'] == 1024).all() and (t['c1'] == 1024).all()
    t = pp.opencv_linear_tables(4, 8, False)         # rows keep the fraction at the border, columns do not
    assert (t['i0'][0], t['i1'][0], t['c0'][0], t['c1'][0]) == (0, 0, 512, 1536)
    t = pp.opencv_linear_tables(4, 8, True)
    assert (t['i0'][0], t['i1'][0], t['c0'][0], t['c1'][0]) == (0, 1, 2048, 0)
    for n_in, n_out in ((0, 5), (5, 0), (-1, 3)):
        with pytest.raises(RuntimeError, match='at least 1'):
            pp.opencv_linear_tables(n_in, n_out)


def test_gpu_preprocess_opencv_flag_follows_the_reference():
    """opencv=True takes the OpenCV path only with fast_rescaling: --precise-rescaling is scipy with OpenCV installed"""
    assert pp.GpuPreprocess(641, batched=True, opencv=True).opencv
    assert not pp.GpuPreprocess(641, batched=True).opencv
    g = pp.GpuPreprocess(641, batched=True, fast_rescaling=False, opencv=True)
    assert not g.opencv and not g.fast_rescaling
    with pytest.raises(RuntimeError, match='only BILINEAR'):
        pp.GpuPreprocess(641, batched=True, opencv=True, resample=3)


@pytest.mark.skipif(torch.cuda.is_available(), reason='only meaningful without a GPU')
def test_abi_without_gpu_returns_cuda_error_and_refuses_bad_arguments():
    """no CPU path: a well-formed call fails at its first CUDA call; a bad one is refused before it"""
    L = _lib.lib()
    descs = (_lib.CvImage * 1)()
    d = descs[0]
    d.src, d.pitch, d.h, d.w, d.th, d.tw, d.left, d.top, d.ytab, d.xtab = 4096, 30, 4, 10, 8, 5, 0, 0, 0, 8
    taps = np.concatenate([pp.opencv_linear_tables(4, 8, False), pp.opencv_linear_tables(10, 5, True)])
    ws_bytes = ctypes.sizeof(descs) + taps.nbytes

    def call(descs=descs, taps=taps):
        return L.pifpaf_image_resize_linear_cv_u8(descs, 1, taps.ctypes.data, taps.size, 8192, ws_bytes, 65536, 8, 5,
                                                  None)
    assert call() == _lib.E_CUDA
    d.pitch = 29
    assert call() == _lib.E_BADARG and b'pitch' in L.pifpaf_last_error()
    d.pitch = 30
    bad = taps.copy()
    bad['c1'][3] += 1                                # 2049 in all: OpenCV's int16 lanes would saturate
    assert call(taps=bad) == _lib.E_BADARG
    bad = taps.copy()
    bad['i1'][9] = 10                                # column 10 of a 10-pixel source
    assert call(taps=bad) == _lib.E_BADARG


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='reference package not staged')
def test_opencv_resize_and_meta_equal_reference_transforms(tmp_path):
    """the reference's own RescaleAbsolute(fast=True) with its module-level cv2 left in place, run in a subprocess:
    Predictor's composition with CenterPad and with CenterPadTight(16)"""
    pytest.importorskip('cv2')
    script = textwrap.dedent('''
        import warnings
        warnings.filterwarnings('ignore')
        import numpy as np, PIL.Image, torch
        import openpifpaf
        from openpifpaf import transforms
        from openpifpaf_b200 import preprocess as pp
        assert transforms.scale.cv2 is not None, 'the reference did not import cv2'

        def mine(img, long_edge, batched, fill):
            h, w = img.shape[:2]
            g = pp.GpuPreprocess.__new__(pp.GpuPreprocess)          # host logic only
            g.long_edge, g.batched, g.multiple = long_edge, batched, 16
            (tw, th, ltrb, (cw, ch)), = g.plan([(w, h)])[0]
            canvas = np.empty((ch, cw, 3), dtype=np.uint8)
            canvas[:] = fill
            canvas[ltrb[1]:ltrb[1] + th, ltrb[0]:ltrb[0] + tw] = pp.opencv_linear_reference(img, tw, th)
            return canvas, pp.reference_meta(w, h, tw, th, np.asarray(ltrb))

        def check(pre, img, long_edge, batched, what):
            torch.manual_seed(3)
            image, _, meta = transforms.Compose(pre)(PIL.Image.fromarray(img), [], None)
            torch.manual_seed(3)
            fill = (int(torch.randint(0, 255, (1,)).item()),) * 3 if batched else pp.TIGHT_PAD_FILL
            canvas, m = mine(img, long_edge, batched, fill)
            assert np.array_equal(np.asarray(image), canvas), (what, img.shape)
            for k in ('offset', 'scale', 'valid_area', 'width_height'):
                assert np.array_equal(np.asarray(meta[k], dtype=np.float64), m[k]), (what, k, meta[k], m[k])

        rng = np.random.default_rng(0)
        shapes = [(427, 640), (480, 360), (390, 427), (429, 427), (27, 28), (1080, 1920), (333, 500), (160, 120)]
        n = 0
        for (h, w) in shapes:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            for le in (641, 321):
                check([transforms.NormalizeAnnotations(), transforms.RescaleAbsolute(le, fast=True),
                       transforms.CenterPad(le)], img, le, True, 'CenterPad')
                check([transforms.NormalizeAnnotations(), transforms.RescaleAbsolute(le, fast=True),
                       transforms.CenterPadTight(16)], img, le, False, 'CenterPadTight')
                n += 1
        print('OPENCV_REF_OK', n)
    ''')
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', script], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=900)
    assert 'OPENCV_REF_OK' in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
