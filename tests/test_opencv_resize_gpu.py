"""GPU: the OpenCV rescale, pifpaf_image_resize_linear_cv_u8 (cv2.resize(INTER_LINEAR) + CenterPad in one launch per
batch), against the stored outputs of cv2 (tests/golden/opencv_resize.npz), the numpy restatement, and cv2 itself
where it is installed.

The C ABI over one mixed batch: the fixture's cases (clamped border rows, an exact 2x reduction, 1-pixel rows,
columns and images, phone photos) plus larger sizes and a source with padded rows.  Inside each window every byte
must equal OpenCV, every pad byte the image's colour, and the bytes beyond the batch's canvases must keep their
sentinels; each image must equal the same image resized alone.  Refused calls write nothing.  Then
`GpuPreprocess(opencv=True)`, `raw_images` / `jpeg_images` with opencv_rescaling=True, and the reference's own
Predictor with OpenCV importable against raw_images."""
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
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'opencv_resize.npz')
BASE, TAIL = 13, 29          # sentinel bytes before and after the canvases
CW = CH = 641
PAD_ROW = 11                 # extra bytes per source row of the pitched case


def sentinel(n):
    return ((np.arange(n) * 37 + 11) % 251).astype(np.uint8)


def fixture_cases():
    """(img, expected window, h, w, th, tw) of every stored case: cv2's output on a seeded input"""
    z = np.load(GOLDEN)
    out = []
    for i, (seed, (h, w, th, tw)) in enumerate(zip(z['seeds'], z['shapes'])):
        img = np.random.default_rng(int(seed)).integers(0, 256, (h, w, 3), dtype=np.uint8)
        out.append((img, z[f'out_{i}'], int(h), int(w), int(th), int(tw)))
    return out


def live_cv2(img, tw, th):
    try:
        import cv2
    except ImportError:
        return None
    return cv2.resize(np.ascontiguousarray(img), (tw, th), interpolation=cv2.INTER_LINEAR)


def batch_cases():
    """(img, want or None, th, tw, left, top, fill, pitch_pad): the fixture plus sizes the fixture cannot store"""
    rng = np.random.default_rng(2)
    out = []
    x, y = 0, 0
    for k, (img, want, h, w, th, tw) in enumerate(fixture_cases()):
        left, top = (k * 37) % (CW - tw + 1), (k * 53) % (CH - th + 1)
        out.append((img, want, th, tw, left, top, (k, 255 - k, 3 * k), PAD_ROW if k % 4 == 1 else 0))
    for (h, w, th, tw, left, top) in ((480, 640, 481, 641, 0, 80), (3024, 4032, 481, 641, 0, 80),
                                      (962, 1282, 481, 641, 0, 80), (390, 427, 585, 641, 0, 28),
                                      (300, 37, 517, 11, 630, 124), (1, 1, 641, 641, 0, 0)):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        out.append((img, None, th, tw, left, top, (x, y, 200), PAD_ROW if h == 390 else 0))
        x, y = x + 40, y + 20
    return out


class CvCall:
    """images and their taps, staged for one pifpaf_image_resize_linear_cv_u8 into a sentinel-framed canvas buffer"""

    def __init__(self, cases):
        self.cases = cases
        self.srcs, tables, self.descs = [], [], (_lib.CvImage * len(cases))()
        n = 0
        for d, (img, _, th, tw, left, top, fill, pad) in zip(self.descs, cases):
            h, w = img.shape[:2]
            rows = np.zeros((h, w * 3 + pad), dtype=np.uint8)
            rows[:, :w * 3] = img.reshape(h, w * 3)
            src = torch.from_numpy(rows).cuda()
            self.srcs.append(src)
            d.src, d.pitch, d.h, d.w, d.th, d.tw, d.left, d.top = src.data_ptr(), w * 3 + pad, h, w, th, tw, left, top
            d.fill[:3] = fill
            d.ytab, d.xtab = n, n + th
            tables += [pp.opencv_linear_tables(h, th, horizontal=False),
                       pp.opencv_linear_tables(w, tw, horizontal=True)]
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
        rc = _lib.lib().pifpaf_image_resize_linear_cv_u8(a['images'], a['n'], a['taps'], a['n_taps'], a['ws'],
                                                         a['ws_bytes'], a['canvas'], a['ch'], a['cw'], None)
        torch.cuda.synchronize()
        return rc, self.buf.cpu().numpy()

    def canvases(self, got):
        return got[BASE:BASE + len(self.cases) * self.plane].reshape(len(self.cases), CH, CW, 3)


@pytest.mark.gpu
def test_cv_abi_mixed_batch_equals_opencv_in_one_launch():
    cases = batch_cases()
    call = CvCall(cases)
    n0 = _lib.lib().pifpaf_launch_count()
    rc, got = call.run()
    assert rc == _lib.OK, _lib.lib().pifpaf_last_error()
    assert _lib.lib().pifpaf_launch_count() - n0 == 1
    assert np.array_equal(got[:BASE], call.before[:BASE]) and np.array_equal(got[-TAIL:], call.before[-TAIL:])
    canv = call.canvases(got)
    live = 0
    for i, (img, stored, th, tw, left, top, fill, pad) in enumerate(cases):
        window = canv[i, top:top + th, left:left + tw]
        wants = [pp.opencv_linear_reference(img, tw, th)] + ([stored] if stored is not None else [])
        cv = live_cv2(img, tw, th)
        if cv is not None:
            wants.append(cv)
            live += 1
        for want in wants:
            bad = np.argwhere(window != want)
            assert bad.size == 0, f'image {i} {img.shape} -> {(th, tw)}: {len(bad)} bytes differ, first at {bad[0]}'
        padmask = np.ones((CH, CW), dtype=bool)
        padmask[top:top + th, left:left + tw] = False
        assert (canv[i][padmask] == np.asarray(fill, dtype=np.uint8)).all(), f'image {i}: pad colour'
    print(f'{len(cases)} images in one launch, {live} also against live cv2')
    for i, case in enumerate(cases):
        alone = CvCall([case])
        rc, g1 = alone.run()
        assert rc == _lib.OK and np.array_equal(alone.canvases(g1)[0], canv[i]), f'image {i} alone'


@pytest.mark.gpu
def test_cv_abi_refusals_write_nothing():
    cases = batch_cases()[:3]
    call = CvCall(cases)
    good = call.descs

    def with_desc(i, **fields):
        d = (_lib.CvImage * len(good))()
        ctypes.memmove(d, good, ctypes.sizeof(good))
        for k, v in fields.items():
            setattr(d[i], k, v)
        return d

    def with_tap(k, **fields):
        t = call.taps.copy()
        for f, v in fields.items():
            t[f][k] = v
        return t
    tw0, th1 = cases[0][3], cases[1][2]
    h1 = cases[1][0].shape[0]
    cases_bad = [
        dict(n=0), dict(images=None), dict(taps=None), dict(n_taps=0), dict(canvas=None), dict(ws=None),
        dict(ch=0), dict(cw=0), dict(ws_bytes=call.ws_bytes - 1), dict(n_taps=call.taps.size - 1),
        dict(images=with_desc(1, src=None)), dict(images=with_desc(1, h=0)), dict(images=with_desc(1, w=-1)),
        dict(images=with_desc(1, th=0)), dict(images=with_desc(1, tw=0)),
        dict(images=with_desc(0, pitch=3 * cases[0][0].shape[1] - 1)),
        dict(images=with_desc(0, left=CW - tw0 + 1)), dict(images=with_desc(1, top=CH - th1 + 1)),
        dict(images=with_desc(1, left=-1)), dict(images=with_desc(1, top=-1)),
        dict(images=with_desc(2, ytab=-1)), dict(images=with_desc(2, xtab=call.taps.size)),
        dict(images=with_desc(1, h=h1 - 1)),                    # taps index a row the source does not have
    ]
    t = with_tap(3, c0=-1, c1=2049)
    cases_bad.append(dict(taps=t.ctypes.data, keep=t))
    t = with_tap(5, c1=call.taps['c1'][5] + 1)                 # sum 2049: OpenCV's int16 lanes would saturate
    cases_bad.append(dict(taps=t.ctypes.data, keep=t))
    t = with_tap(0, i0=-1)
    cases_bad.append(dict(taps=t.ctypes.data, keep=t))
    for o in cases_bad:
        o = {k: v for k, v in o.items() if k != 'keep'}
        rc, got = call.run(**o)
        assert rc == _lib.E_BADARG, (o, rc)
        assert np.array_equal(got, call.before), f'{o}: a refused call wrote'
    rc, got = call.run()
    assert rc == _lib.OK and not np.array_equal(got, call.before)


def reference_compose(img, long_edge, batched, fill, multiple=16):
    """RescaleAbsolute(fast=True) with OpenCV + CenterPad / CenterPadTight: the restatement (cv2 where installed),
    torchvision's pad with the same fill, and the meta of those transforms"""
    PIL = pytest.importorskip('PIL.Image')
    import torchvision.transforms.functional as TF
    img = np.ascontiguousarray(img)
    h, w = img.shape[:2]
    tw, th = pp.rescale_target(w, h, long_edge)
    resized = pp.opencv_linear_reference(img, tw, th)
    cv = live_cv2(img, tw, th)
    if cv is not None:
        assert np.array_equal(cv, resized)
    cw = ch = long_edge
    if not batched:
        cw = (tw - 1 + multiple - 1) // multiple * multiple + 1
        ch = (th - 1 + multiple - 1) // multiple * multiple + 1
    ltrb = pp.center_pad_ltrb(tw, th, cw, ch)
    return (np.asarray(TF.pad(PIL.fromarray(resized), list(ltrb), fill=tuple(fill))),
            pp.reference_meta(w, h, tw, th, np.asarray(ltrb)))


def assert_meta_equal(got, want):
    for k in ('offset', 'scale', 'valid_area', 'width_height'):
        assert np.array_equal(np.asarray(got[k], dtype=np.float64), np.asarray(want[k], dtype=np.float64)), k


@pytest.mark.gpu
def test_gpu_preprocess_opencv_equals_opencv_and_torchvision_pad():
    """host, CUDA and strided inputs; every fill form; CenterPad and CenterPadTight; with fast_rescaling=False the
    scipy path wins"""
    rng = np.random.default_rng(8)
    base = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w) in ((427, 640), (390, 427), (300, 200))]
    big = rng.integers(0, 256, (500, 600, 3), dtype=np.uint8)
    big_cuda = torch.from_numpy(big).cuda()
    images = [base[0], torch.from_numpy(base[1]).cuda(), base[2][..., ::-1], big_cuda[3:3 + 211, 7:7 + 333],
              torch.from_numpy(big)[50:50 + 98, 9:9 + 401]]
    want_imgs = [base[0], base[1], base[2][..., ::-1], big[3:214, 7:340], big[50:148, 9:410]]
    fills = [(11, 12, 13), 22, 33, 44, (0, 255, 1)]
    colours = pp.pad_fills(fills, len(images), True)
    g = pp.GpuPreprocess(641, batched=True, opencv=True)
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
    for fill in (7, (1, 2, 3)):                             # one grey, one colour for every image
        c, _ = g(images[:2], fill=fill)
        for i in range(2):
            want, _ = reference_compose(want_imgs[i], 641, True, pp.pad_fills(fill, 1, True)[0])
            np.testing.assert_array_equal(c[i].cpu().numpy(), want)
    with pytest.raises(RuntimeError, match='out of range'):
        g(images[:1], fill=256)
    # batch size 1: CenterPadTight(16) and its colour
    c1, m1 = pp.GpuPreprocess(385, batched=False, opencv=True)([base[1]])
    want, meta = reference_compose(base[1], 385, False, pp.TIGHT_PAD_FILL)
    np.testing.assert_array_equal(c1[0].cpu().numpy(), want)
    assert_meta_equal(m1[0], meta)
    # --precise-rescaling with OpenCV installed is scipy
    precise, _ = pp.GpuPreprocess(641, batched=True, fast_rescaling=False, opencv=True)(images, fill=fills)
    scipy_canvas, _ = pp.GpuPreprocess(641, batched=True, fast_rescaling=False)(images, fill=fills)
    assert torch.equal(precise, scipy_canvas) and not torch.equal(precise, canvas)


def tiny_predictor(monkeypatch):
    from openpifpaf_b200 import constants, decoder, network, predictor
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=-2.0)
    for hd in plan['heads']:
        hd['w'] = hd['w'] * np.float32(0.06)
    return predictor.Predictor(network.CompiledNet(plan, 161, 161, 2), constants.COCO_N_KEYPOINTS,
                               constants.COCO_PERSON_SKELETON)


@pytest.mark.gpu
def test_jpeg_images_opencv_equal_raw_images_on_pillow_arrays(monkeypatch):
    PIL = pytest.importorskip('PIL.Image')
    rng = np.random.default_rng(3)
    datas = []
    for (h, w) in ((120, 161), (161, 100), (300, 200)):
        buf = io.BytesIO()
        PIL.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(buf, format='JPEG', quality=90)
        datas.append(buf.getvalue())
    arrays = [pp.pillow_rgb(d) for d in datas]
    pred = tiny_predictor(monkeypatch)
    fills = [3, (10, 20, 30), 250]
    want = pred.raw_images(arrays, fill=fills, opencv_rescaling=True)
    got = pred.jpeg_images(datas, fill=fills, opencv_rescaling=True)
    assert sum(d.shape[0] for d, _, _ in want) > 0
    for (d, s, m), (wd, ws, wm) in zip(got, want):
        np.testing.assert_array_equal(d, wd)
        np.testing.assert_array_equal(s, ws)
        assert_meta_equal(m, wm)
    # one preprocess per (fast_rescaling, opencv) path; fast_rescaling=False ignores opencv_rescaling
    pred.raw_images(arrays[:1], fill=3, fast_rescaling=False, opencv_rescaling=True)
    pred.raw_images(arrays[:1], fill=3)
    assert sorted(pred._gpu_preprocess) == [(False, False), (True, False), (True, True)]
    assert pred._gpu_preprocess[(True, True)].opencv and not pred._gpu_preprocess[(True, False)].opencv
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
    torch.ops.openpifpaf.set_quiet(True)
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED
    assert openpifpaf.transforms.scale.cv2 is not None          # the reference rescales with OpenCV

    B = 3
    openpifpaf.Predictor.batch_size = B
    openpifpaf.Predictor.long_edge = 641
    openpifpaf.Predictor.loader_workers = 0
    torch.manual_seed(0)
    openpifpaf.network.Factory.base_name = 'shufflenetv2k16'
    openpifpaf.network.Factory.checkpoint = None
    datamodule = openpifpaf.plugins.coco.CocoKp()
    predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas, json_data=True)
    assert predictor.fast_rescaling
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
    shapes = [(900, 1200), (390, 427), (640, 100), (412, 480), (150, 200), (480, 360), (333, 500)]
    raw = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w) in shapes]
    ref = list(predictor.numpy_images(raw))
    TF.pad = pad
    assert len(ref) == len(raw) and len(recorded) == len(raw), (len(ref), len(recorded))

    mine = b200_predictor.from_shell(model, 641, 641, B)
    got = mine.raw_images(raw, json_data=True, fill=recorded, score_weights=COCO_PERSON_SCORE_WEIGHTS,
                          opencv_rescaling=True)
    n = 0
    for i, ((want, _, wmeta), (js, meta)) in enumerate(zip(ref, got)):
        assert js == want, (i, len(js), len(want))
        for k in ('offset', 'scale', 'valid_area', 'width_height'):
            assert np.array_equal(np.asarray(wmeta[k], dtype=np.float64), meta[k]), (i, k, wmeta[k], meta[k])
        n += len(want)
    assert n > 0
    print('RAW_IMAGES_OPENCV_REF_OK', n, 'poses on', len(raw), 'images, greys', recorded)
''')


@pytest.mark.gpu
def test_raw_images_opencv_equal_reference_predictor_numpy_images(tmp_path):
    """the reference's own Predictor with OpenCV importable (batch size 3, long edge 641, cv2.resize, CenterPad,
    CifCafB200) on 7 images == raw_images(opencv_rescaling=True) with the greys its CenterPad drew"""
    try:
        import cv2          # noqa: F401
    except ImportError:
        pytest.skip('OpenCV is not installed, so the reference rescales with Pillow here')
    if not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')):
        pytest.skip('oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', REFERENCE_SCRIPT], capture_output=True, text=True, env=env,
                       cwd=str(tmp_path), timeout=900)
    assert 'RAW_IMAGES_OPENCV_REF_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout.strip().splitlines()[-1])
