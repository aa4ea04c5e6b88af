"""GPU: the image preprocessing of preprocess.cu on every launch sequence and edge, against Pillow.

`pifpaf_image_resize_bilinear_u8` alone, through the C ABI: each case writes into the middle of a larger canvas
pre-filled with a sentinel byte pattern, at unaligned source and destination addresses.  Inside the target window the
result must equal `PIL.Image.resize(BILINEAR)` and the numpy restatement byte for byte; every byte outside it must keep
its sentinel.  Refused calls must write nothing.  Then `GpuPreprocess` against the reference's composition (Pillow
resize + torchvision's pad with the same fill, `reference_meta`), the uint8 stem on tight non-square canvases,
`Predictor.raw_images` over several batches, and the reference's own `Predictor.numpy_images` against `raw_images`.

`test_cases_reach_every_resize_path` (CPU) checks with `preprocess.resize_path` that the case lists below reach all
five launch sequences."""
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
PATHS = {'hv', 'h_dense', 'h_pitched', 'v', 'copy'}

# (h, w, target_w, target_h, lead, trail): the destination rows start `lead` bytes into a row of pitch
# lead + 3 * target_w + trail bytes (lead = trail = 0 is a dense destination)
ABI_CASES = [
    (427, 640, 321, 214, 9, 12),          # down x down
    (50, 70, 161, 123, 3, 3),             # up x up (3-tap tables)
    (60, 500, 641, 30, 0, 6),             # up x down
    (300, 37, 11, 517, 6, 0),             # down x up
    (33, 100, 257, 33, 0, 0),             # horizontal only, dense, up
    (45, 999, 97, 45, 0, 0),              # horizontal only, dense, down, odd source rows
    (33, 100, 257, 33, 3, 0),             # horizontal only, pitched
    (1, 37, 5, 1, 1, 2),                  # 1 x N -> 1 x 5, pitched at an odd byte
    (100, 33, 33, 257, 3, 9),             # vertical only, up
    (641, 77, 77, 97, 1, 1),              # vertical only, down
    (29, 1, 1, 7, 2, 0),                  # N x 1, vertical only
    (41, 61, 61, 41, 5, 7),               # no rescale, odd row bytes
    (1, 1, 1, 1, 1, 1),                   # no rescale, one pixel
    (1, 1, 13, 11, 4, 0),                 # one pixel -> 13 x 11
    (40, 30, 1, 1, 0, 0),                 # -> one pixel
    (1, 900, 1, 900, 0, 3),               # one row -> one column
    (900, 1, 900, 1, 0, 0),               # one column -> one row
    (3, 25600, 128, 3, 0, 0),             # 200x horizontal reduction: 401 taps
    (20000, 5, 5, 97, 3, 0),              # 206x vertical reduction: 415 taps
    (2000, 3000, 12, 9, 0, 9),            # both directions, 501 and 447 taps
    (3024, 4032, 641, 480, 0, 0),         # phone photo to 641
    (600, 8192, 641, 46, 0, 0),           # panorama to 641
]
TOP, BOTTOM, BASE, TAIL = 2, 3, 5, 7      # sentinel rows above / below the window, bytes before / after the canvas

# GpuPreprocess cases: name -> (long_edge, batched, [(h, w)])
PREPROCESS_CASES = {
    # (h < 640, 640) keeps its height at long edge 641: (100, 640) and (427, 640) take the horizontal-only path
    'batched641': (641, True, [(900, 1200), (100, 640), (640, 100), (641, 300), (150, 200), (427, 640)]),
    'tight400': (400, False, [(100, 399), (97, 390)]),        # 400 wide on a 401-wide canvas: pitched horizontal
    'tight_no_rescale': (None, False, [(100, 200), (99, 196)]),
    'one_pixel_no_rescale': (None, False, [(37, 1)]),
}


def abi_path(case):
    h, w, tw, th, lead, trail = case
    return pp.resize_path(w, h, tw, th, lead + 3 * tw + trail)


def preprocess_paths(long_edge, batched, shapes):
    g = pp.GpuPreprocess.__new__(pp.GpuPreprocess)          # host logic only
    g.long_edge, g.batched, g.multiple = long_edge, batched, 16
    plans, (cw, _) = g.plan([(w, h) for (h, w) in shapes])
    return [pp.resize_path(w, h, tw, th, 3 * cw) for (h, w), (tw, th, _, _) in zip(shapes, plans)]


def test_cases_reach_every_resize_path():
    assert {abi_path(c) for c in ABI_CASES} == PATHS
    assert set().union(*(preprocess_paths(*c) for c in PREPROCESS_CASES.values())) == PATHS
    assert preprocess_paths(*PREPROCESS_CASES['batched641']) == ['hv', 'h_dense', 'v', 'copy', 'hv', 'h_dense']
    assert preprocess_paths(*PREPROCESS_CASES['tight400'])[0] == 'h_pitched'
    assert max(pp.pil_bilinear_coeffs(25600, 128)[1].shape[1], pp.pil_bilinear_coeffs(20000, 97)[1].shape[1]) > 400


# ---------------------------------------------------------------------------------------------------- the C ABI alone
def sentinel(n):
    return ((np.arange(n) * 37 + 11) % 251).astype(np.uint8)


def dev_ptr(t, offset=0):
    return None if t is None else t.data_ptr() + offset


def pil_resize(img, tw, th):
    PIL = pytest.importorskip('PIL.Image')
    return np.asarray(PIL.fromarray(np.ascontiguousarray(img)).resize((tw, th), PIL.BILINEAR))


class AbiCall:
    """One resize of a random [h, w, 3] image into a sentinel-filled canvas through the C ABI."""

    def __init__(self, h, w, tw, th, lead, trail, seed=0):
        self.h, self.w, self.tw, self.th = h, w, tw, th
        self.img = np.random.default_rng(seed + h * 31 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
        self.pitch = lead + 3 * tw + trail
        self.dst_off = BASE + TOP * self.pitch + lead
        self.before = sentinel(BASE + (TOP + th + BOTTOM) * self.pitch + TAIL)
        self.canvas = torch.from_numpy(self.before).cuda()
        src = np.concatenate([sentinel(1), self.img.ravel()])                   # the image starts at an odd address
        self.src = torch.from_numpy(src).cuda()
        self.tables = {}
        for axis, n_in, n_out in (('x', w, tw), ('y', h, th)):
            b, k = pp.pil_bilinear_coeffs(n_in, n_out)
            self.tables[axis] = (torch.from_numpy(b).cuda(), torch.from_numpy(k).cuda(), k.shape[1])
        self.tmp = torch.empty((h * tw * 3 + 1,), dtype=torch.uint8, device='cuda')

    def run(self, **override):
        a = dict(src=dev_ptr(self.src, 1), h=self.h, w=self.w, dst=dev_ptr(self.canvas, self.dst_off), pitch=self.pitch,
                 th=self.th, tw=self.tw, xb=dev_ptr(self.tables['x'][0]), xk=dev_ptr(self.tables['x'][1]),
                 xks=self.tables['x'][2], yb=dev_ptr(self.tables['y'][0]), yk=dev_ptr(self.tables['y'][1]),
                 yks=self.tables['y'][2], tmp=dev_ptr(self.tmp, 1))
        a.update(override)
        rc = _lib.lib().pifpaf_image_resize_bilinear_u8(a['src'], a['h'], a['w'], a['dst'], a['pitch'], a['th'], a['tw'],
                                                         a['xb'], a['xk'], a['xks'], a['yb'], a['yk'], a['yks'],
                                                         a['tmp'], None)
        torch.cuda.synchronize()
        return rc, self.canvas.cpu().numpy()

    def expected(self, window):
        out = self.before.copy()
        for y in range(self.th):
            o = self.dst_off + y * self.pitch
            out[o:o + 3 * self.tw] = window[y].ravel()
        return out


def case_id(c):
    return '%s-%dx%d-to-%dx%d-lead%d-trail%d' % ((abi_path(c),) + c)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ABI_CASES, ids=case_id)
def test_resize_abi_equals_pillow_inside_the_window_and_nothing_outside(case):
    call = AbiCall(*case)
    want = pil_resize(call.img, call.tw, call.th)
    np.testing.assert_array_equal(pp.resize_bilinear_reference(call.img, call.tw, call.th), want)
    rc, got = call.run()
    assert rc == _lib.OK, _lib.lib().pifpaf_last_error()
    exp = call.expected(want)
    bad = np.flatnonzero(got != exp)
    assert bad.size == 0, (f'{bad.size} bytes differ, first at canvas byte {bad[0]} '
                           f'(window starts at {call.dst_off}, pitch {call.pitch})')


@pytest.mark.gpu
def test_resize_abi_refusals_write_nothing():
    hv = AbiCall(50, 70, 161, 123, 3, 3)            # needs both tables and tmp
    hp = AbiCall(33, 100, 257, 33, 3, 0)            # horizontal only, pitched: needs tmp
    v = AbiCall(100, 33, 33, 257, 3, 9)             # vertical only
    cases = [
        (hv, dict(h=0)), (hv, dict(w=0)), (hv, dict(th=0)), (hv, dict(tw=0)), (hv, dict(h=-3)),
        (hv, dict(src=None)), (hv, dict(dst=None)),
        (hv, dict(pitch=161 * 3 - 1)), (hp, dict(pitch=257 * 3 - 1)), (v, dict(pitch=0)),
        (hv, dict(xb=None)), (hv, dict(xk=None)), (hv, dict(xks=0)),
        (hv, dict(yb=None)), (hv, dict(yk=None)), (hv, dict(yks=0)),
        (hp, dict(xb=None)), (hp, dict(xks=0)), (v, dict(yk=None)), (v, dict(yks=0)),
        (hv, dict(tmp=None)), (hp, dict(tmp=None)),
    ]
    for call, override in cases:
        rc, got = call.run(**override)
        assert rc == _lib.E_BADARG, (override, rc)
        assert np.array_equal(got, call.before), f'{override}: a refused call wrote to the canvas'
    # what is not needed may be absent: the vertical path without x tables or tmp, a copy without any table
    rc, got = v.run(xb=None, xk=None, xks=0, tmp=None)
    assert rc == _lib.OK and np.array_equal(got, v.expected(pil_resize(v.img, v.tw, v.th)))
    cp = AbiCall(41, 61, 61, 41, 5, 7)
    rc, got = cp.run(xb=None, xk=None, xks=0, yb=None, yk=None, yks=0, tmp=None)
    assert rc == _lib.OK and np.array_equal(got, cp.expected(cp.img))


@pytest.mark.gpu
def test_fill_rgb_abi():
    L = _lib.lib()
    before = sentinel(64)
    buf = torch.from_numpy(before).cuda()
    p = buf.data_ptr() + 7                          # odd start

    def fill(n, r, g, b, ptr=p):
        rc = L.pifpaf_image_fill_rgb(ptr, n, r, g, b, None)
        torch.cuda.synchronize()
        return rc, buf.cpu().numpy()

    rc, got = fill(0, 1, 2, 3)
    assert rc == _lib.OK and np.array_equal(got, before)
    for n, r, g, b, ptr in ((3, -1, 0, 0, p), (3, 0, 256, 0, p), (3, 0, 0, 300, p), (3, 0, 0, -7, p), (-1, 1, 2, 3, p),
                            (3, 1, 2, 3, None)):
        rc, got = fill(n, r, g, b, ptr)
        assert rc == _lib.E_BADARG and np.array_equal(got, before), (n, r, g, b, ptr)
    rc, got = fill(5, 0, 128, 255)
    want = before.copy()
    want[7:22] = np.tile([0, 128, 255], 5)
    assert rc == _lib.OK and np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------- GpuPreprocess
def reference_compose(img, long_edge, batched, fill, multiple=16):
    """the reference's RescaleAbsolute (Pillow path) + CenterPad / CenterPadTight: PIL resize, torchvision's pad with
    the same fill, and the meta of those transforms"""
    PIL = pytest.importorskip('PIL.Image')
    import torchvision.transforms.functional as TF
    h, w = img.shape[:2]
    im = PIL.fromarray(np.ascontiguousarray(img))
    tw, th = (w, h)
    if long_edge:
        tw, th = pp.rescale_target(w, h, long_edge)
        im = im.resize((tw, th), PIL.BILINEAR)
    if batched:
        cw = ch = long_edge
    else:
        cw = (tw - 1 + multiple - 1) // multiple * multiple + 1
        ch = (th - 1 + multiple - 1) // multiple * multiple + 1
    ltrb = pp.center_pad_ltrb(tw, th, cw, ch)
    canvas = np.asarray(TF.pad(im, list(ltrb), fill=tuple(fill)))
    assert canvas.shape == (ch, cw, 3)
    return canvas, pp.reference_meta(w, h, tw, th, np.asarray(ltrb), rescaled=long_edge is not None)


def assert_meta_equal(got, want):
    for k in ('offset', 'scale', 'valid_area', 'width_height'):
        assert np.array_equal(np.asarray(got[k], dtype=np.float64), np.asarray(want[k], dtype=np.float64)), (k, got[k], want[k])
    assert got['hflip'] == want['hflip'] and got['rotation'] == want['rotation']


def random_images(shapes, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w) in shapes]


def check_preprocess(g, images, fill, want_fills):
    """g(images, fill) == reference_compose of each image with its own colour"""
    canvas, metas = g(images, fill=fill)
    got = canvas.cpu().numpy()
    assert len(metas) == len(images) == got.shape[0]
    for i, (img, f) in enumerate(zip(images, want_fills)):
        host = img.cpu().numpy() if isinstance(img, torch.Tensor) else np.asarray(img)
        want, meta = reference_compose(host, g.long_edge, g.batched, f)
        assert got[i].shape == want.shape
        bad = np.argwhere(got[i] != want)
        assert bad.size == 0, f'image {i} {host.shape}: {len(bad)} bytes differ, first at {bad[0]}'
        assert_meta_equal(metas[i], meta)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(PREPROCESS_CASES))
def test_gpu_preprocess_equals_pillow_and_torchvision_pad(name):
    long_edge, batched, shapes = PREPROCESS_CASES[name]
    images = random_images(shapes, seed=len(name))
    g = pp.GpuPreprocess(long_edge, batched=batched)
    if batched:
        fills = [(i * 53 % 256, 255 - i, 7 * i) for i in range(len(images))]
        check_preprocess(g, images, fills, fills)
    else:
        check_preprocess(g, images, None, [pp.TIGHT_PAD_FILL] * len(images))


@pytest.mark.gpu
def test_gpu_preprocess_fill_forms():
    """an int is a grey for every image, a tuple one colour for every image (also at B = 3), a list per image"""
    images = random_images([(120, 161), (161, 100), (70, 90)], seed=3)
    g = pp.GpuPreprocess(161, batched=True)
    check_preprocess(g, images, 9, [(9, 9, 9)] * 3)
    check_preprocess(g, images, (10, 200, 30), [(10, 200, 30)] * 3)
    check_preprocess(g, images[:2], (10, 200, 30), [(10, 200, 30)] * 2)
    check_preprocess(g, images, [0, (1, 2, 3), 255], [(0, 0, 0), (1, 2, 3), (255, 255, 255)])
    with pytest.raises(RuntimeError, match='colours for'):
        g(images, fill=[1, 2])
    with pytest.raises(RuntimeError, match='out of range'):
        g(images, fill=256)


@pytest.mark.gpu
def test_gpu_preprocess_cuda_and_strided_inputs():
    """CUDA-resident images, a BGR -> RGB view img[..., ::-1], and non-contiguous host and CUDA views equal the
    contiguous host images"""
    rng = np.random.default_rng(8)
    base = random_images([(427, 640), (300, 200), (150, 161)], seed=8)
    big = rng.integers(0, 256, (400, 500, 3), dtype=np.uint8)
    big_cuda = torch.from_numpy(big).cuda()
    images = [torch.from_numpy(base[0]).cuda(),                         # CUDA, contiguous
              base[1][..., ::-1],                                        # BGR view, negative stride
              big_cuda[3:3 + 211, 7:7 + 333],                            # CUDA, row-strided view
              torch.from_numpy(big)[50:50 + 98, 9:9 + 401],              # host tensor, row-strided view
              base[2]]
    want_imgs = [base[0], np.ascontiguousarray(base[1][..., ::-1]), big[3:3 + 211, 7:7 + 333], big[50:148, 9:410],
                 base[2]]
    g = pp.GpuPreprocess(641, batched=True)
    fills = [11, 22, 33, 44, 55]
    canvas, metas = g(images, fill=fills)
    got = canvas.cpu().numpy()
    for i, (img, f) in enumerate(zip(want_imgs, fills)):
        want, meta = reference_compose(img, 641, True, (f, f, f))
        np.testing.assert_array_equal(got[i], want, err_msg=f'image {i}')
        assert_meta_equal(metas[i], meta)
    # on a stream other than the one the CUDA images were written on
    side = torch.cuda.Stream()
    canvas2, _ = g(images, fill=fills, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(canvas2, canvas)


@pytest.mark.gpu
def test_gpu_preprocess_refusals():
    g = pp.GpuPreprocess(None, batched=False)
    with pytest.raises(RuntimeError, match='share the padded size'):
        g(random_images([(100, 200), (100, 300)], seed=1))
    with pytest.raises(RuntimeError, match='uint8'):
        g([np.zeros((10, 10, 3), dtype=np.float32)])
    with pytest.raises(RuntimeError, match='uint8'):
        g([np.zeros((10, 10, 4), dtype=np.uint8)])
    with pytest.raises(RuntimeError, match='long-edge'):
        pp.GpuPreprocess(None, batched=True)


# ---------------------------------------------------------------------------------------------------- uint8 stem
@pytest.mark.gpu
@pytest.mark.parametrize('H,W,shapes', [(257, 401, [(250, 395), (240, 380)]), (401, 161, [(395, 150), (390, 147)])],
                         ids=['257x401', '401x161'])
def test_uint8_stem_on_tight_canvases_equals_float_stem(H, W, shapes):
    """GpuPreprocess(CenterPadTight) canvas -> forward_uint8 == forward on the host-normalised Pillow canvas, bit for
    bit, on non-square tight canvases"""
    from openpifpaf_b200 import network
    images = random_images(shapes, seed=H)
    g = pp.GpuPreprocess(max(H, W), batched=False)
    canvas, _ = g(images)
    assert tuple(canvas.shape) == (2, H, W, 3)
    want = [reference_compose(img, max(H, W), False, pp.TIGHT_PAD_FILL)[0] for img in images]
    assert np.array_equal(canvas.cpu().numpy(), np.stack(want))
    net = network.CompiledNet(network.random_plan('shufflenetv2k16', seed=2, confidence_bias=0.0), H, W, 2)
    heads_u8 = [t.clone() for t in net.forward_uint8(canvas)]
    x = normalise(np.stack(want)).cuda()
    for a, b in zip(heads_u8, net.forward(x)):
        assert torch.isfinite(a).all() and torch.equal(a, b)
    net.close()


def normalise(canvases):
    """ToTensor + Normalize of the reference's EVAL_TRANSFORM on uint8 [B, H, W, 3] host canvases"""
    from openpifpaf_b200 import network
    mean = torch.tensor(network.CompiledNet.IMAGE_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(network.CompiledNet.IMAGE_STD).view(1, 3, 1, 1)
    return (torch.from_numpy(canvases).permute(0, 3, 1, 2).float().div(255.0) - mean) / std


# ---------------------------------------------------------------------------------------------------- raw_images
@pytest.mark.gpu
def test_raw_images_over_several_batches_equal_batch_on_reference_canvases(monkeypatch):
    """2 * max_batch + 1 images with one pad colour each: raw_images == Predictor.batch on each batch of
    reference-composed, host-normalised canvases followed by inverse_transform_batch; overlap_decode changes nothing"""
    from openpifpaf_b200 import constants, decoder, network, predictor
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)     # keep the random-init poses
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=-2.0)
    for hd in plan['heads']:
        hd['w'] = hd['w'] * np.float32(0.06)
    S, MB = 161, 2
    shapes = [(120, 161), (161, 100), (300, 200), (90, 250), (161, 161)]
    images = random_images(shapes, seed=21)
    fills = [3, (10, 20, 30), 250, 77, (0, 128, 255)]
    colours = pp.pad_fills(fills, len(images), True)
    # the API takes CUDA images and BGR views too
    api_images = list(images)
    api_images[1] = torch.from_numpy(images[1]).cuda()
    api_images[3] = np.ascontiguousarray(images[3][..., ::-1])[..., ::-1]

    composed = [reference_compose(img, S, True, c) for img, c in zip(images, colours)]
    pred = predictor.Predictor(network.CompiledNet(plan, S, S, MB), constants.COCO_N_KEYPOINTS,
                               constants.COCO_PERSON_SKELETON)
    want = []
    for i in range(0, len(images), MB):
        x = normalise(np.stack([c for c, _ in composed[i:i + MB]])).pin_memory()
        for (ann, _), (_, meta) in zip(pred.batch(x), composed[i:i + MB]):
            want.append(pp.inverse_transform_batch(ann.numpy(), meta))
    assert sum(d.shape[0] for d, _ in want) > 0

    got = pred.raw_images(api_images, fill=fills)
    assert len(got) == len(images)
    for i, ((data, scales, meta), (wd, ws), (_, wmeta)) in enumerate(zip(got, want, composed)):
        np.testing.assert_array_equal(data, wd, err_msg=f'image {i}')
        np.testing.assert_array_equal(scales, ws, err_msg=f'image {i}')
        assert_meta_equal(meta, wmeta)
    weights = np.linspace(3.0, 1.0, constants.COCO_N_KEYPOINTS)
    js = pred.raw_images(api_images, fill=fills, json_data=True, score_weights=weights)
    for (j, _), (wd, ws) in zip(js, want):
        assert j == pp.json_data_batch(wd, ws, score_weights=weights)
    pred.close()

    ovl = predictor.Predictor(network.CompiledNet(plan, S, S, MB), constants.COCO_N_KEYPOINTS,
                              constants.COCO_PERSON_SKELETON, overlap_decode=True)
    for (data, scales, _), (wd, ws) in zip(ovl.raw_images(api_images, fill=fills), want):
        np.testing.assert_array_equal(data, wd)
        np.testing.assert_array_equal(scales, ws)
    ovl.close()


# ---------------------------------------------------------------------------------------------------- the reference
REFERENCE_SCRIPT = textwrap.dedent('''
    import sys, warnings
    warnings.filterwarnings('ignore')
    import numpy as np
    import torch
    import torchvision.transforms.functional as TF
    import openpifpaf
    import openpifpaf.transforms.scale as scale_mod
    from openpifpaf.plugins.coco.constants import COCO_PERSON_SCORE_WEIGHTS
    from openpifpaf_b200 import predictor as b200_predictor
    torch.ops.openpifpaf.set_quiet(True)
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED
    scale_mod.cv2 = None                                    # the Pillow path of RescaleAbsolute (transforms/scale.py:56-59)

    B = 3
    openpifpaf.Predictor.batch_size = B
    openpifpaf.Predictor.long_edge = 641
    openpifpaf.Predictor.loader_workers = 0
    torch.manual_seed(0)
    openpifpaf.network.Factory.base_name = 'shufflenetv2k16'
    openpifpaf.network.Factory.checkpoint = None
    datamodule = openpifpaf.plugins.coco.CocoKp()
    predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas, json_data=True)
    assert type(predictor.processor.decoders[0]).__name__ == 'CifCafB200'
    model = predictor.model_cpu
    # trained-network-like head statistics (as in test_plugin_gpu.py), and every seed completed into a pose
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

    recorded = []                                           # the grey CenterPad draws for each image, in order
    pad = TF.pad
    def recording_pad(img, padding, fill=0, padding_mode='constant'):
        recorded.append(tuple(int(c) for c in fill))
        return pad(img, padding, fill=fill, padding_mode=padding_mode)
    TF.pad = recording_pad

    rng = np.random.default_rng(5)
    shapes = [(900, 1200), (100, 640), (640, 100), (641, 300), (150, 200), (480, 360), (333, 500)]
    raw = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w) in shapes]
    ref = list(predictor.numpy_images(raw))
    TF.pad = pad
    assert len(ref) == len(raw) and len(recorded) == len(raw), (len(ref), len(recorded))

    mine = b200_predictor.from_shell(model, 641, 641, B)
    got = mine.raw_images(raw, json_data=True, fill=recorded, score_weights=COCO_PERSON_SCORE_WEIGHTS)
    n = 0
    for i, ((want, _, wmeta), (js, meta)) in enumerate(zip(ref, got)):
        assert js == want, (i, len(js), len(want))
        for k in ('offset', 'scale', 'valid_area', 'width_height'):
            assert np.array_equal(np.asarray(wmeta[k], dtype=np.float64), meta[k]), (i, k, wmeta[k], meta[k])
        n += len(want)
    assert n > 0
    print('RAW_IMAGES_REF_OK', n, 'poses on', len(raw), 'images, greys', recorded)
''')


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
def test_raw_images_equal_reference_predictor_numpy_images(tmp_path):
    """the reference's own Predictor (batch size 3, long edge 641, Pillow rescale, CenterPad, CifCafB200) on 7 images
    == raw_images with the greys its CenterPad drew: the same json dicts, image for image"""
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', REFERENCE_SCRIPT], capture_output=True, text=True, env=env,
                       cwd=str(tmp_path), timeout=900)
    assert 'RAW_IMAGES_REF_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout.strip().splitlines()[-1])
