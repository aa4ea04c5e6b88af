"""CPU: the batches of Predictor.raw_images(tight_pad=True) -- images grouped by their CenterPadTight(16) canvas, at most
max_batch per batch, input order kept -- and their canvases and metas against the reference's own
Compose([NormalizeAnnotations, RescaleAbsolute, CenterPadTight(16)]) on mixed aspect ratios."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from openpifpaf_b200 import predictor
from openpifpaf_b200 import preprocess as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')

# (w, h): landscape, portrait, square, panorama, tiny and odd photo sizes
SIZES = [(640, 480), (480, 640), (500, 375), (640, 480), (375, 500), (800, 600), (333, 500), (640, 427), (1280, 720),
         (640, 480), (50, 50), (1, 37), (640, 480), (481, 641), (427, 640), (2000, 1000)]


def canvas_of(w, h, long_edge):
    g = pp.GpuPreprocess.__new__(pp.GpuPreprocess)          # host logic only
    g.long_edge, g.batched, g.multiple = long_edge, False, 16
    (_, _, _, (cw, ch)), = g.plan([(w, h)])[0]
    return ch, cw


@pytest.mark.parametrize('long_edge', [641, 321, None])
@pytest.mark.parametrize('max_batch', [1, 2, 3, 64])
def test_groups_cover_every_image_once_in_order(long_edge, max_batch):
    sizes = SIZES if long_edge else SIZES[:11]
    groups = predictor.tight_pad_groups(sizes, long_edge, max_batch, (2001, 2001))
    seen = [i for _, idx in groups for i in idx]
    assert sorted(seen) == list(range(len(sizes)))
    firsts = []
    for canvas, idx in groups:
        assert 1 <= len(idx) <= max_batch and idx == sorted(idx)
        assert all(canvas_of(*sizes[i], long_edge) == canvas for i in idx)
        if canvas not in [c for c, _ in firsts]:
            firsts.append((canvas, idx[0]))
    assert [i for _, i in firsts] == sorted(i for _, i in firsts)        # canvases in order of their first image
    # each canvas's images fill whole batches before the next batch of that canvas starts
    for canvas in {c for c, _ in groups}:
        lens = [len(idx) for c, idx in groups if c == canvas]
        assert all(n == max_batch for n in lens[:-1])


def test_a_canvas_above_capacity_is_refused():
    assert predictor.tight_pad_groups([(640, 480)], 641, 4, (481, 641))
    for cap in ((480, 641), (481, 640)):
        with pytest.raises(RuntimeError, match='above the net'):
            predictor.tight_pad_groups([(640, 480), (640, 480)], 641, 4, cap)
    with pytest.raises(RuntimeError, match='image 1'):
        predictor.tight_pad_groups([(640, 480), (480, 640)], 641, 4, (481, 641))


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')), reason='reference package not staged')
def test_canvases_and_metas_equal_reference_compose(tmp_path):
    """the reference's NormalizeAnnotations -> RescaleAbsolute -> CenterPadTight(16) on mixed aspect ratios gives the
    canvas of each image's group and the meta raw_images returns (reference_meta of GpuPreprocess's plan)"""
    script = textwrap.dedent('''
        import numpy as np, PIL.Image
        from openpifpaf import transforms
        import openpifpaf.transforms.scale as scale_mod
        scale_mod.cv2 = None
        from openpifpaf_b200 import predictor, preprocess as pp
        SIZES = %r
        for long_edge in (641, 321, None):
            sizes = SIZES if long_edge else SIZES[:11]
            groups = predictor.tight_pad_groups(sizes, long_edge, 3, (2001, 2001))
            canvas_of = {i: c for c, idx in groups for i in idx}
            g = pp.GpuPreprocess.__new__(pp.GpuPreprocess)
            g.long_edge, g.batched, g.multiple = long_edge, False, 16
            for i, (w, h) in enumerate(sizes):
                if long_edge and min(w, h) == 1:
                    continue                                # _scale divides by zero there, in both
                pre = [transforms.NormalizeAnnotations()]
                if long_edge:
                    pre.append(transforms.RescaleAbsolute(long_edge, fast=True))
                pre.append(transforms.CenterPadTight(16))
                img = PIL.Image.fromarray(np.zeros((h, w, 3), dtype=np.uint8))
                image, _, meta = transforms.Compose(pre)(img, [], None)
                assert image.size[::-1] == canvas_of[i], (i, image.size, canvas_of[i])
                (tw, th, ltrb, _), = g.plan([(w, h)])[0]
                mine = pp.reference_meta(w, h, tw, th, np.asarray(ltrb), rescaled=long_edge is not None)
                for k in ('offset', 'scale', 'valid_area', 'width_height'):
                    assert np.array_equal(np.asarray(meta[k], dtype=np.float64), mine[k]), (i, k, meta[k], mine[k])
        print('TIGHT_PAD_REF_OK')
    ''' % (SIZES,))
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', script], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=600)
    assert 'TIGHT_PAD_REF_OK' in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
