"""CPU: the precise rescale (transforms.RescaleAbsolute(fast=False) -> scipy.ndimage.zoom(order=1),
transforms/scale.py:60-67) restated by `preprocess.scipy_zoom_tables` / `zoom_linear_reference`, against scipy itself
on a seeded size sweep that must contain both of scipy's quirks (a cval last row or column, and a sample textbook
bilinear rounds differently), and against the reference's own transforms when the staged reference package exists."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from openpifpaf_b200 import preprocess as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')

# (w, h) of common photos, rescaled as RescaleAbsolute would for the long edges below
PHOTO_SIZES = [(640, 480), (480, 640), (640, 427), (427, 640), (500, 375), (375, 500), (612, 612), (800, 600),
               (1024, 768), (1280, 720), (1920, 1080), (4032, 3024), (3024, 4032), (640, 360), (333, 500), (28, 27)]
LONG_EDGES = (321, 641, 801)


def sweep_sizes(n=340, seed=0):
    """(h, w, target_w, target_h): n random sizes in 1..900 (up, down and mixed), 1-pixel rows, columns, inputs and
    outputs, and every RescaleAbsolute target of PHOTO_SIZES at LONG_EDGES"""
    rng = np.random.default_rng(seed)
    out = [tuple(int(v) for v in rng.integers(1, 901, 4)) for _ in range(n)]
    out += [(1, int(w), int(tw), 1) for w, tw in rng.integers(1, 901, (3, 2))]           # 1 x N -> 1 x M
    out += [(int(h), 1, 1, int(th)) for h, th in rng.integers(1, 901, (3, 2))]           # N x 1 -> M x 1
    out += [(1, 1, 1, 1), (1, 1, 13, 11), (1, 37, 5, 1), (29, 1, 1, 7), (40, 30, 1, 1), (1, 900, 1, 900),
            (900, 1, 900, 1), (27, 28, 27, 28), (28, 27, 28, 27), (2, 2, 900, 3), (900, 900, 1, 2)]
    for le in LONG_EDGES:
        out += [(h, w) + pp.rescale_target(w, h, le) for (w, h) in PHOTO_SIZES]
    return out


def scipy_zoom(img, tw, th):
    import scipy.ndimage
    h, w = img.shape[:2]
    return scipy.ndimage.zoom(img, (th / h, tw / w, 1), order=1)


def textbook_bilinear(img, tw, th):
    """float64 bilinear at scipy's sample positions, lerped x then y and rounded half to even (numpy.rint)"""
    h, w = img.shape[:2]

    def axis(n_in, n_out):
        cc = np.arange(n_out) * ((n_in - 1) / (n_out - 1) if n_out != 1 else 1.0)
        i0 = np.minimum(np.floor(cc).astype(np.int64), n_in - 1)
        return i0, np.minimum(i0 + 1, n_in - 1), cc - i0
    y0, y1, fy = axis(h, th)
    x0, x1, fx = axis(w, tw)
    v = img.astype(np.float64)
    fx, fy = fx[None, :, None], fy[:, None, None]
    top = v[y0][:, x0] * (1 - fx) + v[y0][:, x1] * fx
    bot = v[y1][:, x0] * (1 - fx) + v[y1][:, x1] * fx
    return np.clip(np.rint(top * (1 - fy) + bot * fy), 0, 255).astype(np.uint8)


def test_zoom_restatement_equals_scipy_on_a_sweep():
    scipy = pytest.importorskip('scipy')
    print('scipy', scipy.__version__)
    rng = np.random.default_rng(23)
    sizes = sweep_sizes()
    assert len(sizes) >= 400
    bad, cval_edges, rounding = [], 0, 0
    for (h, w, tw, th) in sizes:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        want = scipy_zoom(img, tw, th)
        got = pp.zoom_linear_reference(img, tw, th)
        if got.shape != want.shape or not np.array_equal(got, want):
            bad.append((h, w, tw, th))
            continue
        outside_y = pp.scipy_zoom_tables(h, th)['i0'] < 0
        outside_x = pp.scipy_zoom_tables(w, tw)['i0'] < 0
        if outside_y.any() or outside_x.any():
            cval_edges += 1
            assert (want[outside_y] == 0).all() and (want[:, outside_x] == 0).all()
        inside = ~outside_y[:, None] & ~outside_x[None, :]
        rounding += int((textbook_bilinear(img, tw, th) != want)[inside].sum())
    assert not bad, f'{len(bad)} sizes differ from scipy, first: {bad[:5]}'
    print(f'{len(sizes)} sizes, {cval_edges} with a cval row or column, {rounding} samples textbook bilinear rounds '
          'differently')
    assert cval_edges >= 1 and rounding >= 1


def test_zoom_tables_on_degenerate_sizes():
    t = pp.scipy_zoom_tables(28, 27)                     # 26 * (27 / 26) = 27.000000000000004 > 27: cval
    assert t['i0'][-1] == -1 and (t['i0'][:-1] >= 0).all()
    t = pp.scipy_zoom_tables(27, 28)                     # 27 * (26 / 27) lands on 26 exactly: inside
    assert (t['i0'] >= 0).all() and t['i0'][-1] == 26 and t['w1'][-1] == 0.0
    t = pp.scipy_zoom_tables(1, 5)                       # one input sample: zoom 0, every output reads it
    assert (t['i0'] == 0).all() and (t['i1'] == 0).all() and (t['w0'] == 1.0).all() and (t['w1'] == 0.0).all()
    t = pp.scipy_zoom_tables(37, 1)                      # one output sample: zoom_div 0 -> zoom 1, reads input 0
    assert (t['i0'], t['i1'], t['w0'], t['w1']) == (0, 1, 1.0, 0.0)
    t = pp.scipy_zoom_tables(1, 1)
    assert (t['i0'], t['i1'], t['w0'], t['w1']) == (0, 0, 1.0, 0.0)
    t = pp.scipy_zoom_tables(50, 50)                     # unchanged: the identity
    assert np.array_equal(t['i0'], np.arange(50)) and (t['w0'] == 1.0).all() and (t['w1'] == 0.0).all()
    t = pp.scipy_zoom_tables(640, 641)
    assert t.dtype.itemsize == 24 and (t['i1'] <= 639).all() and (t['i1'][t['i0'] >= 0] >= t['i0'][t['i0'] >= 0]).all()
    for n_in, n_out in ((0, 5), (5, 0), (-1, 3)):
        with pytest.raises(RuntimeError, match='at least 1'):
            pp.scipy_zoom_tables(n_in, n_out)


def test_only_bilinear_is_built():
    for resample in (0, 3, 1, 'bilinear'):
        with pytest.raises(RuntimeError, match='only BILINEAR'):
            pp.GpuPreprocess(641, batched=True, fast_rescaling=False, resample=resample)
        with pytest.raises(RuntimeError, match='only BILINEAR'):
            pp.GpuPreprocess(641, batched=True, resample=resample)
    g = pp.GpuPreprocess(641, batched=True, fast_rescaling=False, resample=pp.BILINEAR)
    assert not g.fast_rescaling and pp.GpuPreprocess(641, batched=True).fast_rescaling


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')), reason='reference package not staged')
def test_zoom_and_meta_equal_reference_transforms(tmp_path):
    """the reference's own transforms with the scipy rescale, run in a subprocess: Predictor's composition with
    CenterPad and with CenterPadTight(16), and CocoKp.common_eval_preprocess at batch size 1 and 4"""
    script = textwrap.dedent('''
        import warnings
        warnings.filterwarnings('ignore')
        import numpy as np, PIL.Image, torch
        import openpifpaf
        from openpifpaf import transforms
        from openpifpaf.plugins.coco import CocoKp
        from openpifpaf_b200 import preprocess as pp

        def mine(img, long_edge, batched, fill):
            h, w = img.shape[:2]
            g = pp.GpuPreprocess.__new__(pp.GpuPreprocess)          # host logic only
            g.long_edge, g.batched, g.multiple = long_edge, batched, 16
            (tw, th, ltrb, (cw, ch)), = g.plan([(w, h)])[0]
            canvas = np.empty((ch, cw, 3), dtype=np.uint8)
            canvas[:] = fill
            canvas[ltrb[1]:ltrb[1] + th, ltrb[0]:ltrb[0] + tw] = pp.zoom_linear_reference(img, tw, th)
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
        shapes = [(427, 640), (480, 360), (390, 427), (429, 427), (27, 28), (1080, 1920), (333, 500)]
        n = 0
        for (h, w) in shapes:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            for le in (641, 321):
                check([transforms.NormalizeAnnotations(), transforms.RescaleAbsolute(le, fast=False),
                       transforms.CenterPad(le)], img, le, True, 'CenterPad')
                check([transforms.NormalizeAnnotations(), transforms.RescaleAbsolute(le, fast=False),
                       transforms.CenterPadTight(16)], img, le, False, 'CenterPadTight')
                for bs in (1, 4):
                    CocoKp.eval_long_edge, CocoKp.batch_size = le, bs
                    pre = [t for t in CocoKp.common_eval_preprocess() if t is not None]
                    check(pre, img, le, bs > 1, f'common_eval_preprocess batch {bs}')
                n += 1
        print('ZOOM_REF_OK', n)
    ''')
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', script], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=900)
    assert 'ZOOM_REF_OK' in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
