"""Image preprocessing (SURVEY.md 8f rank 2).

CPU: the restatement of Pillow's ImagingResample (coefficient tables + integer arithmetic) against PIL.Image.resize
itself -- Pillow is the third-party dependency the reference resizes with (transforms/scale.py:56-59); the meta dicts
and the batched inverse_transform / json_data against the reference's own transforms / Annotation (when the staged
reference package exists).  GPU: the kernels against PIL + torchvision's pad, and the whole raw-image path."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from openpifpaf_b200 import preprocess as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')

SIZES = [(480, 640, 641, 481), (375, 500, 321, 241), (100, 37, 161, 435), (600, 800, 400, 300), (33, 33, 33, 65),
         (720, 1280, 641, 360), (50, 50, 50, 50), (427, 640, 640, 427), (2, 3, 7, 5), (1080, 1920, 321, 180)]


@pytest.mark.parametrize('h,w,tw,th', SIZES)
def test_pillow_bilinear_restatement_is_bit_exact(h, w, tw, th):
    PIL = pytest.importorskip('PIL.Image')
    img = np.random.default_rng(h * 7 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    want = np.asarray(PIL.fromarray(img).resize((tw, th), PIL.BILINEAR))
    np.testing.assert_array_equal(pp.resize_bilinear_reference(img, tw, th), want)


def sweep_sizes(n=300, seed=0):
    """n random (h, w, target_w, target_h) in 1..900 -- up, down, mixed and unchanged directions -- followed by the
    edges: 1-pixel rows and columns, 200x reductions (401 taps), a phone photo and a panorama to 641"""
    rng = np.random.default_rng(seed)
    out = [tuple(int(v) for v in rng.integers(1, 901, 4)) for _ in range(n)]
    out += [(h, w, w, th) for (h, w, th) in rng.integers(1, 901, (4, 3)).tolist()]        # vertical only
    out += [(h, w, tw, h) for (h, w, tw) in rng.integers(1, 901, (4, 3)).tolist()]        # horizontal only
    return out + [(1, 1, 1, 1), (1, 1, 13, 11), (1, 37, 5, 1), (1, 37, 37, 9), (29, 1, 1, 7), (40, 30, 1, 1),
                  (1, 900, 1, 900), (900, 1, 900, 1), (3, 25600, 128, 3), (20000, 5, 5, 97), (3024, 4032, 641, 480),
                  (600, 8192, 641, 46)]


def test_pillow_bilinear_restatement_random_sweep():
    """the numpy restatement == PIL.Image.resize(BILINEAR) byte for byte on every size of `sweep_sizes`"""
    PIL = pytest.importorskip('PIL.Image')
    rng = np.random.default_rng(17)
    bad = []
    for (h, w, tw, th) in sweep_sizes():
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        want = np.asarray(PIL.fromarray(img).resize((tw, th), PIL.BILINEAR))
        got = pp.resize_bilinear_reference(img, tw, th)
        if got.shape != want.shape or not np.array_equal(got, want):
            bad.append((h, w, tw, th))
    assert not bad, f'{len(bad)} sizes differ from Pillow, first: {bad[:5]}'


def test_pad_fills_tuple_is_one_colour_list_is_per_image():
    assert pp.pad_fills((1, 2, 3), 3, True) == [(1, 2, 3)] * 3            # not three greys at B = 3
    assert pp.pad_fills((1, 2, 3), 2, True) == [(1, 2, 3)] * 2
    assert pp.pad_fills(7, 3, True) == [(7, 7, 7)] * 3
    assert pp.pad_fills(np.uint8(9), 1, True) == [(9, 9, 9)]
    assert pp.pad_fills([5, (1, 2, 3), np.array([4, 5, 6])], 3, True) == [(5, 5, 5), (1, 2, 3), (4, 5, 6)]
    assert pp.pad_fills([(1, 2, 3)], 1, True) == [(1, 2, 3)]
    for fill, n in (([1, 2], 3), ([1, 2, 3], 2), ([(1, 2, 3)], 3), ([], 1)):
        with pytest.raises(RuntimeError, match='colours for'):
            pp.pad_fills(fill, n, True)
    for fill in ((1, 2), [(1, 2, 3, 4)]):
        with pytest.raises(RuntimeError, match='triple'):
            pp.pad_fills(fill, 1, True)
    # default: CenterPad draws one torch.randint(0, 255) grey per image in order, CenterPadTight a fixed colour
    torch.manual_seed(4)
    greys = [int(torch.randint(0, 255, (1,)).item()) for _ in range(3)]
    torch.manual_seed(4)
    assert pp.pad_fills(None, 3, True) == [(g, g, g) for g in greys]
    assert pp.pad_fills(None, 2, False) == [pp.TIGHT_PAD_FILL] * 2


def test_raw_image_chunks_slice_per_image_fills():
    """Predictor.raw_images pads image i with fill[i] in every batch of max_batch images, not fill[i % max_batch]"""
    from openpifpaf_b200 import predictor
    images = [f'image{i}' for i in range(7)]
    fills = [(i, 2 * i, 3 * i) for i in range(7)]
    chunks = list(predictor.raw_image_chunks(images, 3, fills))
    assert [c for c, _ in chunks] == [images[0:3], images[3:6], images[6:7]]
    assert [f for _, f in chunks] == [fills[0:3], fills[3:6], fills[6:7]]
    for fill in (None, 5, (1, 2, 3)):
        assert [f for _, f in predictor.raw_image_chunks(images, 3, fill)] == [fill] * 3
    assert [c for c, _ in predictor.raw_image_chunks(images, 7, None)] == [images]
    with pytest.raises(RuntimeError, match='colours for'):
        list(predictor.raw_image_chunks(images, 3, fills[:3]))


def test_reference_meta_without_rescale_on_one_pixel_images():
    """no long edge: RescaleAbsolute is not in the pipeline, so a 1-pixel-wide or -high image has no scale factor
    (the reference never divides by w - 1); with a long edge the reference's _scale divides by zero, and so does this"""
    for (w, h) in ((1, 37), (50, 1), (1, 1)):
        g = pp.GpuPreprocess.__new__(pp.GpuPreprocess)
        g.long_edge, g.batched, g.multiple = None, False, 16
        (tw, th, ltrb, _), = g.plan([(w, h)])[0]
        meta = pp.reference_meta(w, h, tw, th, np.asarray(ltrb), rescaled=False)
        assert np.array_equal(meta['scale'], (1.0, 1.0)) and np.array_equal(meta['offset'], (-ltrb[0], -ltrb[1]))
        assert np.array_equal(meta['valid_area'], (ltrb[0], ltrb[1], w - 1, h - 1))
        with pytest.raises(ZeroDivisionError):
            pp.reference_meta(w, h, *pp.rescale_target(w, h, 161), np.asarray(ltrb))
    # two-pixel images keep their factors, and a size the rescale leaves unchanged has factors of exactly 1
    meta = pp.reference_meta(2, 3, 5, 7, np.zeros(4), rescaled=True)
    assert np.array_equal(meta['scale'], (4.0, 3.0))
    assert np.array_equal(pp.reference_meta(300, 641, 300, 641, np.zeros(4))['scale'], (1.0, 1.0))


def test_coefficient_tables_are_normalised():
    for n_in, n_out in ((640, 641), (1280, 321), (37, 161)):
        bounds, kk = pp.pil_bilinear_coeffs(n_in, n_out)
        assert bounds.shape == (n_out, 2) and (bounds[:, 0] >= 0).all() and (bounds[:, 0] + bounds[:, 1] <= n_in).all()
        assert np.abs(kk.sum(axis=1) - (1 << pp.PRECISION_BITS)).max() <= kk.shape[1]      # rounding of each tap


def test_inverse_transform_and_json_batch_forms():
    """array forms == per-annotation arithmetic of annotation.py:121-214, written out (numpy-2 roundings)"""
    rng = np.random.default_rng(1)
    ann = rng.random((5, 17, 4)).astype(np.float32) * np.array([1, 600, 400, 9], dtype=np.float32)
    ann[2, 3:9, 0] = 0.0
    meta = pp.reference_meta(640, 427, 641, 428, np.asarray(pp.center_pad_ltrb(641, 428, 641, 641)))
    data, scales = pp.inverse_transform_batch(ann, meta)
    for i in range(5):
        d = np.stack([ann[i, :, 1], ann[i, :, 2], ann[i, :, 0]], axis=1).astype(np.float32)
        d[:, 0] += meta['offset'][0]
        d[:, 1] += meta['offset'][1]
        d[:, 0] = d[:, 0] / meta['scale'][0]
        d[:, 1] = d[:, 1] / meta['scale'][1]
        s = ann[i, :, 3].copy()
        s /= meta['scale'][0]
        np.testing.assert_array_equal(data[i], d)
        np.testing.assert_array_equal(scales[i], s)
    js = pp.json_data_batch(data, scales)
    assert len(js) == 5 and len(js[0]['keypoints']) == 51 and js[0]['score'] >= 0.001


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')), reason='reference package not staged')
def test_meta_and_annotations_equal_reference_transforms(tmp_path):
    """the reference's own Predictor preprocessing (PIL path) and Annotation methods, run in a subprocess"""
    script = textwrap.dedent('''
        import sys, warnings
        warnings.filterwarnings('ignore')
        import numpy as np, PIL.Image, torch
        import openpifpaf
        from openpifpaf import transforms
        import openpifpaf.transforms.scale as scale_mod
        scale_mod.cv2 = None                         # the documented Pillow path (transforms/scale.py:56-59)
        from openpifpaf_b200 import preprocess as pp
        from openpifpaf.plugins.coco.constants import COCO_KEYPOINTS, COCO_PERSON_SKELETON, COCO_PERSON_SCORE_WEIGHTS
        rng = np.random.default_rng(0)
        for (h, w, long_edge, batched) in ((427, 640, 641, True), (480, 360, 321, True), (333, 500, 385, False),
                                           (200, 300, None, False), (37, 1, None, False), (1, 50, None, False),
                                           (1, 1, None, False), (37, 1, 161, True), (1, 50, 161, False)):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            pre = [transforms.NormalizeAnnotations()]
            if long_edge:
                pre.append(transforms.RescaleAbsolute(long_edge, fast=True))
            pre.append(transforms.CenterPad(long_edge) if batched else transforms.CenterPadTight(16))
            torch.manual_seed(3)
            if long_edge and min(h, w) == 1:
                # _scale divides by w - 1 or h - 1: the reference and reference_meta both refuse the image
                for fn in (lambda: transforms.Compose(pre)(PIL.Image.fromarray(img), [], None),
                           lambda: pp.reference_meta(w, h, *pp.rescale_target(w, h, long_edge), np.zeros(4))):
                    try:
                        fn()
                        raise AssertionError(('no ZeroDivisionError', h, w))
                    except ZeroDivisionError:
                        pass
                continue
            image, anns, meta = transforms.Compose(pre)(PIL.Image.fromarray(img), [], None)
            torch.manual_seed(3)
            fill = int(torch.randint(0, 255, (1,)).item())
            g = pp.GpuPreprocess.__new__(pp.GpuPreprocess)          # host logic only (no GPU here)
            g.long_edge, g.batched, g.multiple = long_edge, batched, 16
            (tw, th, ltrb, (cw, ch)), = g.plan([(w, h)])[0]
            assert image.size == (cw, ch), (image.size, cw, ch)
            canvas = np.empty((ch, cw, 3), dtype=np.uint8)
            canvas[:] = (fill, fill, fill) if batched else pp.TIGHT_PAD_FILL
            canvas[ltrb[1]:ltrb[1] + th, ltrb[0]:ltrb[0] + tw] = pp.resize_bilinear_reference(img, tw, th)
            assert np.array_equal(np.asarray(image), canvas), 'resized + padded image differs'
            mine = pp.reference_meta(w, h, tw, th, np.asarray(ltrb), rescaled=long_edge is not None)
            for k in ('offset', 'scale', 'valid_area', 'width_height'):
                assert np.array_equal(np.asarray(meta[k], dtype=np.float64), np.asarray(mine[k], dtype=np.float64)), (k, meta[k], mine[k])
            # annotations: inverse_transform + json_data
            dec = rng.random((4, 17, 4)).astype(np.float32) * np.array([1, cw, ch, 9], dtype=np.float32)
            dec[1, 5:11, 0] = 0.0
            data, scales = pp.inverse_transform_batch(dec, mine)
            js = pp.json_data_batch(data, scales, score_weights=COCO_PERSON_SCORE_WEIGHTS)
            for i in range(4):
                a = openpifpaf.Annotation(COCO_KEYPOINTS, COCO_PERSON_SKELETON, score_weights=COCO_PERSON_SCORE_WEIGHTS)
                a.data[:, :2] = dec[i, :, 1:3]; a.data[:, 2] = dec[i, :, 0]; a.joint_scales[:] = dec[i, :, 3]
                b = a.inverse_transform(meta)
                assert np.array_equal(b.data, data[i]) and np.array_equal(b.joint_scales, scales[i])
                assert b.json_data() == js[i], (b.json_data(), js[i])
        print('PREPROCESS_REF_OK')
    ''')
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', script], capture_output=True, text=True, env=env, cwd=str(tmp_path), timeout=600)
    assert 'PREPROCESS_REF_OK' in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.gpu
def test_gpu_resize_pad_equals_pillow_and_torchvision_pad():
    PIL = pytest.importorskip('PIL.Image')
    rng = np.random.default_rng(5)
    raw = [rng.integers(0, 256, s, dtype=np.uint8) for s in ((427, 640, 3), (640, 480, 3), (641, 641, 3), (90, 1000, 3), (641, 300, 3))]
    fills = [7, 200, 0, 33, 255]
    g = pp.GpuPreprocess(641, batched=True)
    canvas, metas = g(raw, fill=fills)
    assert tuple(canvas.shape) == (5, 641, 641, 3)
    got = canvas.cpu().numpy()
    for i, (img, fill) in enumerate(zip(raw, fills)):
        h, w = img.shape[:2]
        tw, th = pp.rescale_target(w, h, 641)
        l, t, _, _ = pp.center_pad_ltrb(tw, th, 641, 641)
        want = np.full((641, 641, 3), fill, dtype=np.uint8)
        want[t:t + th, l:l + tw] = np.asarray(PIL.fromarray(img).resize((tw, th), PIL.BILINEAR))
        np.testing.assert_array_equal(got[i], want)
        assert metas[i]['offset'][0] == -l + 0.0 and metas[i]['scale'][0] == (tw - 1) / (w - 1)
    # batch size 1: CenterPadTight(16)
    g1 = pp.GpuPreprocess(385, batched=False)
    canvas, metas = g1([raw[0]])
    tw, th = pp.rescale_target(640, 427, 385)
    assert tuple(canvas.shape) == (1, (th - 1 + 15) // 16 * 16 + 1, 385, 3)
    l, t, _, _ = pp.center_pad_ltrb(tw, th, 385, canvas.shape[1])
    want = np.empty(tuple(canvas.shape[1:]), dtype=np.uint8)
    want[:] = pp.TIGHT_PAD_FILL                                      # transforms/pad.py:100-101
    want[t:t + th, l:l + tw] = np.asarray(PIL.fromarray(raw[0]).resize((tw, th), PIL.BILINEAR))
    np.testing.assert_array_equal(canvas[0].cpu().numpy(), want)


@pytest.mark.gpu
def test_raw_images_through_preprocess_stem_and_decoder():
    """raw uint8 images -> GPU resize / pad -> uint8 stem -> heads == the reference's PIL + float pipeline fed to the
    float stem, bit for bit; annotations inverse-transformed in one batch"""
    PIL = pytest.importorskip('PIL.Image')
    from openpifpaf_b200 import constants, network, predictor
    rng = np.random.default_rng(11)
    raw = [rng.integers(0, 256, s, dtype=np.uint8) for s in ((120, 161, 3), (161, 100, 3))]
    g = pp.GpuPreprocess(161, batched=True)
    canvas, metas = g(raw, fill=[5, 6])
    plan = network.random_plan('shufflenetv2k16', seed=2, confidence_bias=0.0)
    net = network.CompiledNet(plan, 161, 161, 2)
    heads_u8 = [t.clone() for t in net.forward_uint8(canvas)]
    mean = torch.tensor(network.CompiledNet.IMAGE_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(network.CompiledNet.IMAGE_STD).view(1, 3, 1, 1)
    ref_imgs = []
    for img, fill in zip(raw, (5, 6)):
        h, w = img.shape[:2]
        tw, th = pp.rescale_target(w, h, 161)
        l, t, _, _ = pp.center_pad_ltrb(tw, th, 161, 161)
        c = np.full((161, 161, 3), fill, dtype=np.uint8)
        c[t:t + th, l:l + tw] = np.asarray(PIL.fromarray(img).resize((tw, th), PIL.BILINEAR))
        ref_imgs.append(torch.from_numpy(c).permute(2, 0, 1).float().div(255.0))
    x = ((torch.stack(ref_imgs) - mean) / std).cuda()
    for a, b in zip(heads_u8, net.forward(x)):
        assert torch.equal(a, b)
    pred = predictor.Predictor(net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    res = pred.batch(canvas.cpu().pin_memory())
    via_api = pred.raw_images(raw, fill=[5, 6])
    for (ann, _), meta, (data2, scales2, meta2) in zip(res, metas, via_api):
        data, scales = pp.inverse_transform_batch(ann.numpy(), meta)
        assert data.shape == (ann.shape[0], 17, 3) and np.isfinite(data).all()
        np.testing.assert_array_equal(data, data2)
        np.testing.assert_array_equal(scales, scales2)
    js = pred.raw_images(raw, fill=[5, 6], json_data=True)
    assert len(js) == 2 and all(isinstance(j, list) for j, _ in js)
