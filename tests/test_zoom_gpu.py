"""GPU: the precise rescale, pifpaf_image_zoom_linear_u8 (scipy.ndimage.zoom(order=1) + CenterPad in one launch per
batch), against scipy itself.

The C ABI over one mixed batch: sizes with a cval edge, up and down scaling, per-image colours and a phone photo.
Inside each window every byte must equal scipy, every pad byte the image's colour, and the bytes beyond the batch's
canvases must keep their sentinels; each image must equal the same image resized alone.  Refused calls write nothing.
Then `GpuPreprocess(fast_rescaling=False)` against scipy + torchvision's pad, `raw_images` / `jpeg_images` with
fast_rescaling=False, and the reference's own Predictor with fast_rescaling = False against raw_images."""
import ctypes
import io
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
BASE, TAIL = 13, 29          # sentinel bytes before and after the canvases

# (h, w, target_w, target_h, left, top, fill) on a 641 x 641 canvas
BATCH = [
    (480, 640, 641, 481, 0, 80, (7, 8, 9)),          # up, the flagship size
    (390, 427, 641, 585, 0, 28, (200, 0, 100)),     # RescaleAbsolute(641) target with a black last row
    (28, 28, 27, 27, 300, 2, (1, 2, 3)),            # 28 -> 27 both ways: a black last row and column
    (27, 28, 27, 27, 614, 614, (255, 255, 255)),    # columns 28 -> 27 (black last column), rows unchanged; corner
    (3024, 4032, 641, 480, 0, 80, (33, 66, 99)),    # phone photo, down
    (1, 37, 5, 1, 10, 10, (0, 0, 0)),               # 1 x N
    (29, 1, 1, 7, 20, 20, (90, 91, 92)),            # N x 1
    (1, 1, 13, 11, 30, 40, (5, 5, 5)),              # one pixel -> 13 x 11
    (40, 30, 1, 1, 640, 640, (6, 6, 6)),            # -> one pixel
    (300, 37, 11, 517, 100, 50, (17, 34, 51)),      # down x up
]
CW = CH = 641


def sentinel(n):
    return ((np.arange(n) * 37 + 11) % 251).astype(np.uint8)


def scipy_zoom(img, tw, th):
    import scipy.ndimage
    h, w = img.shape[:2]
    return scipy.ndimage.zoom(img, (th / h, tw / w, 1), order=1)


class ZoomCall:
    """images and their taps, staged for one pifpaf_image_zoom_linear_u8 into a sentinel-framed canvas buffer"""

    def __init__(self, cases, seed=0):
        rng = np.random.default_rng(seed)
        self.cases = cases
        self.imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w, *_) in cases]
        self.srcs = [torch.from_numpy(im).cuda() for im in self.imgs]
        tables, self.descs = [], (_lib.ZoomImage * len(cases))()
        n = 0
        for d, src, (h, w, tw, th, left, top, fill) in zip(self.descs, self.srcs, cases):
            d.src, d.h, d.w, d.th, d.tw, d.left, d.top = src.data_ptr(), h, w, th, tw, left, top
            d.fill[:3] = fill
            d.ytab, d.xtab = n, n + th
            tables += [pp.scipy_zoom_tables(h, th), pp.scipy_zoom_tables(w, tw)]
            n += th + tw
        self.taps = np.concatenate(tables)
        self.plane = CH * CW * 3
        self.before = sentinel(BASE + len(cases) * self.plane + TAIL)
        self.buf = torch.from_numpy(self.before).cuda()
        self.ws_bytes = ctypes.sizeof(self.descs) + self.taps.nbytes
        self.ws = torch.empty((self.ws_bytes,), dtype=torch.uint8, device='cuda')

    def run(self, **o):
        a = dict(images=self.descs, n=len(self.cases), taps=self.taps.ctypes.data, n_taps=self.taps.size,
                 ws=self.ws.data_ptr(), ws_bytes=self.ws_bytes, canvas=self.buf.data_ptr() + BASE, ch=CH, cw=CW)
        a.update(o)
        rc = _lib.lib().pifpaf_image_zoom_linear_u8(a['images'], a['n'], a['taps'], a['n_taps'], a['ws'], a['ws_bytes'],
                                                    a['canvas'], a['ch'], a['cw'], None)
        torch.cuda.synchronize()
        return rc, self.buf.cpu().numpy()

    def canvases(self, got):
        return got[BASE:BASE + len(self.cases) * self.plane].reshape(len(self.cases), CH, CW, 3)


@pytest.mark.gpu
def test_zoom_abi_mixed_batch_equals_scipy_in_one_launch():
    call = ZoomCall(BATCH)
    n0 = _lib.lib().pifpaf_launch_count()
    rc, got = call.run()
    assert rc == _lib.OK, _lib.lib().pifpaf_last_error()
    assert _lib.lib().pifpaf_launch_count() - n0 == 1
    assert np.array_equal(got[:BASE], call.before[:BASE]) and np.array_equal(got[-TAIL:], call.before[-TAIL:])
    canv = call.canvases(got)
    black = 0
    for i, (img, (h, w, tw, th, left, top, fill)) in enumerate(zip(call.imgs, BATCH)):
        want = scipy_zoom(img, tw, th)
        assert want.shape == (th, tw, 3)
        black += int(((pp.scipy_zoom_tables(h, th)['i0'] < 0).any() or (pp.scipy_zoom_tables(w, tw)['i0'] < 0).any()))
        window = canv[i, top:top + th, left:left + tw]
        bad = np.argwhere(window != want)
        assert bad.size == 0, f'image {i} {(h, w, tw, th)}: {len(bad)} bytes differ from scipy, first at {bad[0]}'
        pad = np.ones((CH, CW), dtype=bool)
        pad[top:top + th, left:left + tw] = False
        assert (canv[i][pad] == np.asarray(fill, dtype=np.uint8)).all(), f'image {i}: pad colour'
    assert black >= 2
    # each image alone equals its slot of the batch
    for i, case in enumerate(BATCH):
        alone = ZoomCall([case])
        alone.imgs[0] = call.imgs[i]
        alone.srcs[0].copy_(call.srcs[i])
        rc, g1 = alone.run()
        assert rc == _lib.OK and np.array_equal(alone.canvases(g1)[0], canv[i]), f'image {i} alone'


@pytest.mark.gpu
def test_zoom_abi_refusals_write_nothing():
    call = ZoomCall(BATCH[:3], seed=1)
    good = call.descs

    def with_desc(i, **fields):
        d = (_lib.ZoomImage * len(good))()
        ctypes.memmove(d, good, ctypes.sizeof(good))
        for k, v in fields.items():
            setattr(d[i], k, v)
        return d
    h, w, tw, th = BATCH[1][:4]
    cases = [
        dict(n=0), dict(images=None), dict(taps=None), dict(n_taps=0), dict(canvas=None), dict(ws=None),
        dict(ch=0), dict(cw=0), dict(ws_bytes=call.ws_bytes - 1), dict(n_taps=call.taps.size - 1),
        dict(images=with_desc(1, src=None)), dict(images=with_desc(1, h=0)), dict(images=with_desc(1, w=-1)),
        dict(images=with_desc(1, th=0)), dict(images=with_desc(1, tw=0)),
        dict(images=with_desc(1, left=1)), dict(images=with_desc(1, top=CH - th + 1)),
        dict(images=with_desc(1, left=-1)), dict(images=with_desc(1, top=-1)),
        dict(images=with_desc(2, ytab=-1)), dict(images=with_desc(2, xtab=call.taps.size)),
        dict(images=with_desc(1, h=h - 1)),                         # taps index a row the source does not have
        dict(images=with_desc(0, w=2)),
    ]
    for o in cases:
        rc, got = call.run(**o)
        assert rc == _lib.E_BADARG, (o, rc)
        assert np.array_equal(got, call.before), f'{o}: a refused call wrote'
    rc, got = call.run()
    assert rc == _lib.OK and not np.array_equal(got, call.before)


def reference_compose(img, long_edge, batched, fill, multiple=16):
    """RescaleAbsolute(fast=False) + CenterPad / CenterPadTight: scipy.ndimage.zoom, torchvision's pad with the same
    fill, and the meta of those transforms"""
    PIL = pytest.importorskip('PIL.Image')
    import torchvision.transforms.functional as TF
    h, w = img.shape[:2]
    tw, th = pp.rescale_target(w, h, long_edge)
    im = PIL.fromarray(scipy_zoom(np.ascontiguousarray(img), tw, th))
    cw = ch = long_edge
    if not batched:
        cw = (tw - 1 + multiple - 1) // multiple * multiple + 1
        ch = (th - 1 + multiple - 1) // multiple * multiple + 1
    ltrb = pp.center_pad_ltrb(tw, th, cw, ch)
    return np.asarray(TF.pad(im, list(ltrb), fill=tuple(fill))), pp.reference_meta(w, h, tw, th, np.asarray(ltrb))


def assert_meta_equal(got, want):
    for k in ('offset', 'scale', 'valid_area', 'width_height'):
        assert np.array_equal(np.asarray(got[k], dtype=np.float64), np.asarray(want[k], dtype=np.float64)), k


@pytest.mark.gpu
def test_gpu_preprocess_precise_equals_scipy_and_torchvision_pad():
    """host, CUDA and strided inputs; CenterPad and CenterPadTight; fast_rescaling=True still equals Pillow"""
    PIL = pytest.importorskip('PIL.Image')
    rng = np.random.default_rng(8)
    base = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w) in ((427, 640), (390, 427), (300, 200))]
    big = rng.integers(0, 256, (500, 600, 3), dtype=np.uint8)
    big_cuda = torch.from_numpy(big).cuda()
    images = [base[0], torch.from_numpy(base[1]).cuda(), base[2][..., ::-1], big_cuda[3:3 + 211, 7:7 + 333],
              torch.from_numpy(big)[50:50 + 98, 9:9 + 401]]
    want_imgs = [base[0], base[1], np.ascontiguousarray(base[2][..., ::-1]), big[3:214, 7:340], big[50:148, 9:410]]
    fills = [(11, 12, 13), 22, 33, 44, (0, 255, 1)]
    colours = pp.pad_fills(fills, len(images), True)
    g = pp.GpuPreprocess(641, batched=True, fast_rescaling=False)
    canvas, metas = g(images, fill=fills)
    got = canvas.cpu().numpy()
    for i, (img, c) in enumerate(zip(want_imgs, colours)):
        want, meta = reference_compose(img, 641, True, c)
        np.testing.assert_array_equal(got[i], want, err_msg=f'image {i}')
        assert_meta_equal(metas[i], meta)
    side = torch.cuda.Stream()
    canvas2, _ = g(images, fill=fills, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(canvas2, canvas)
    with pytest.raises(RuntimeError, match='out of range'):
        g(images[:1], fill=256)
    # batch size 1: CenterPadTight(16) and its colour
    g1 = pp.GpuPreprocess(385, batched=False, fast_rescaling=False)
    c1, m1 = g1([base[1]])
    want, meta = reference_compose(base[1], 385, False, pp.TIGHT_PAD_FILL)
    np.testing.assert_array_equal(c1[0].cpu().numpy(), want)
    assert_meta_equal(m1[0], meta)
    # the Pillow path is unchanged
    fast, fmetas = pp.GpuPreprocess(641, batched=True)(images, fill=fills)
    for i, (img, c) in enumerate(zip(want_imgs, colours)):
        tw, th = pp.rescale_target(img.shape[1], img.shape[0], 641)
        l, t, _, _ = pp.center_pad_ltrb(tw, th, 641, 641)
        want = np.empty((641, 641, 3), dtype=np.uint8)
        want[:] = c
        want[t:t + th, l:l + tw] = np.asarray(PIL.fromarray(img).resize((tw, th), PIL.BILINEAR))
        np.testing.assert_array_equal(fast[i].cpu().numpy(), want)
        assert_meta_equal(fmetas[i], metas[i])


@pytest.mark.gpu
def test_jpeg_images_precise_equal_raw_images_on_pillow_arrays(monkeypatch):
    PIL = pytest.importorskip('PIL.Image')
    from openpifpaf_b200 import constants, decoder, network, predictor
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=-2.0)
    for hd in plan['heads']:
        hd['w'] = hd['w'] * np.float32(0.06)
    rng = np.random.default_rng(3)
    datas = []
    for (h, w) in ((120, 161), (161, 100), (300, 200)):
        buf = io.BytesIO()
        PIL.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(buf, format='JPEG', quality=90)
        datas.append(buf.getvalue())
    arrays = [pp.pillow_rgb(d) for d in datas]
    pred = predictor.Predictor(network.CompiledNet(plan, 161, 161, 2), constants.COCO_N_KEYPOINTS,
                               constants.COCO_PERSON_SKELETON)
    fills = [3, (10, 20, 30), 250]
    want = pred.raw_images(arrays, fill=fills, fast_rescaling=False)
    got = pred.jpeg_images(datas, fill=fills, fast_rescaling=False)
    assert sum(d.shape[0] for d, _, _ in want) > 0
    for (d, s, m), (wd, ws, wm) in zip(got, want):
        np.testing.assert_array_equal(d, wd)
        np.testing.assert_array_equal(s, ws)
        assert_meta_equal(m, wm)
    pred.close()


REFERENCE_SCRIPT = textwrap.dedent('''
    import sys, warnings
    warnings.filterwarnings('ignore')
    import numpy as np
    import torch
    import torchvision.transforms.functional as TF
    import openpifpaf
    from openpifpaf.plugins.coco.constants import COCO_PERSON_SCORE_WEIGHTS
    from openpifpaf_b200 import predictor as b200_predictor
    from openpifpaf_b200 import preprocess as pp
    torch.ops.openpifpaf.set_quiet(True)
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED

    B = 3
    openpifpaf.Predictor.batch_size = B
    openpifpaf.Predictor.long_edge = 641
    openpifpaf.Predictor.loader_workers = 0
    openpifpaf.Predictor.fast_rescaling = False              # --precise-rescaling: scipy.ndimage.zoom
    torch.manual_seed(0)
    openpifpaf.network.Factory.base_name = 'shufflenetv2k16'
    openpifpaf.network.Factory.checkpoint = None
    datamodule = openpifpaf.plugins.coco.CocoKp()
    predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas, json_data=True)
    assert type(predictor.processor.decoders[0]).__name__ == 'CifCafB200'
    model = predictor.model_cpu
    with torch.no_grad():
        probe = torch.randn(2, 3, 161, 193, generator=torch.Generator().manual_seed(7)).to(predictor.device)
        feat = model.base_net(probe)
        mu = feat.mean((0, 2, 3))
        std = (feat - mu[None, :, None, None]).pow(2).mean().sqrt()
        for head in model.head_nets:
            w = head.conv.weight / std
            head.conv.bias.copy_(head.conv.bias - w[:, :, 0, 0] @ mu)
            head.conv.weight.copy_(w)
            head.conv.bias.view(head.meta.n_fields, head.n_components, head.upsample_stride ** 2)[:, 1] += -1.0
    import argparse
    parser = argparse.ArgumentParser()
    openpifpaf.decoder.cli(parser)
    openpifpaf.decoder.configure(parser.parse_args(['--force-complete-pose', '--seed-threshold=0.1']))

    recorded = []
    pad = TF.pad
    def recording_pad(img, padding, fill=0, padding_mode='constant'):
        recorded.append(tuple(int(c) for c in fill))
        return pad(img, padding, fill=fill, padding_mode=padding_mode)
    TF.pad = recording_pad

    rng = np.random.default_rng(5)
    # (390, 427) and (412, 480) rescale to 641 wide with a black last row
    shapes = [(900, 1200), (390, 427), (640, 100), (412, 480), (150, 200), (480, 360), (333, 500)]
    black = sum(int((pp.scipy_zoom_tables(h, pp.rescale_target(w, h, 641)[1])['i0'] < 0).any()) for (h, w) in shapes)
    assert black >= 2, black
    raw = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w) in shapes]
    ref = list(predictor.numpy_images(raw))
    TF.pad = pad
    assert len(ref) == len(raw) and len(recorded) == len(raw), (len(ref), len(recorded))

    mine = b200_predictor.from_shell(model, 641, 641, B)
    got = mine.raw_images(raw, json_data=True, fill=recorded, score_weights=COCO_PERSON_SCORE_WEIGHTS,
                          fast_rescaling=False)
    n = 0
    for i, ((want, _, wmeta), (js, meta)) in enumerate(zip(ref, got)):
        assert js == want, (i, len(js), len(want))
        for k in ('offset', 'scale', 'valid_area', 'width_height'):
            assert np.array_equal(np.asarray(wmeta[k], dtype=np.float64), meta[k]), (i, k, wmeta[k], meta[k])
        n += len(want)
    assert n > 0
    print('RAW_IMAGES_PRECISE_REF_OK', n, 'poses on', len(raw), 'images, greys', recorded)
''')


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
def test_raw_images_precise_equal_reference_predictor_numpy_images(tmp_path):
    """the reference's own Predictor with fast_rescaling = False (batch size 3, long edge 641, scipy rescale,
    CenterPad, CifCafB200) on 7 images, two of them with a black edge row == raw_images(fast_rescaling=False) with
    the greys its CenterPad drew"""
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', REFERENCE_SCRIPT], capture_output=True, text=True, env=env,
                       cwd=str(tmp_path), timeout=900)
    assert 'RAW_IMAGES_PRECISE_REF_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout.strip().splitlines()[-1])
