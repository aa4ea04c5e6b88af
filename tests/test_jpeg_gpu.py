"""GPU: pifpaf_jpeg_decode / preprocess.GpuJpegDecoder decode bit-identically to PIL.Image.open(f).convert('RGB')
(the reference's datasets/image_list.py:18) -- a mixed batch of the CPU corpus, a 4032 x 3024 photo, every round cap
of the self-synchronising Huffman decode; Pillow-route streams equal Pillow; malformed streams raise before anything
is written and the handle decodes the next batch; Predictor.jpeg_images equals raw_images on Pillow's arrays and the
reference's own Predictor.images on the same files."""
import io
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from openpifpaf_b200 import preprocess as pp
from openpifpaf_b200 import synth
import jpeg_ref as jr
from test_jpeg import CORPUS, all_ones_huffman, encode, pillow, swapped_scan_order, without

PIL = pytest.importorskip('PIL.Image')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')


def corpus():
    return [encode(h, w, seed=i, **opts) for i, (h, w, opts) in enumerate(CORPUS)]


def pillow_only():
    img = PIL.fromarray(synth.photo_like_image(37, 53, 9))
    out = []
    for kw in (dict(progressive=True), dict(progressive=True, subsampling=0)):
        b = io.BytesIO()
        img.save(b, 'JPEG', quality=85, **kw)
        out.append(b.getvalue())
    b = io.BytesIO()
    img.convert('CMYK').save(b, 'JPEG', quality=90)
    out.append(b.getvalue())
    data = encode(29, 31, seed=4, quality=90, subsampling=0)
    out.append(data[:2] + b'\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00' + data[2:])   # Adobe RGB
    out.append(without(encode(33, 45, seed=5, quality=85, subsampling=2), b'\xff\xc4'))       # standard tables
    return out


def expected_stats(datas, cap):
    """(rounds, fallbacks) of the Python restatement of the self-synchronising decode with the kernels' 1024-bit
    subsequences: rounds that decoded something (the most of any image), serial re-decodes (summed)"""
    rounds = fallbacks = 0
    for d in datas:
        route, hdr = jr.parse(d)
        if route != 'gpu':
            continue
        buf, starts = jr.unstuff(d, hdr['seg'])
        _, r, f = jr.self_sync(hdr, buf, starts, 1024, 16 if cap < 0 else cap)
        rounds, fallbacks = max(rounds, r), fallbacks + f
    return rounds, fallbacks


def assert_equal_pillow(images, datas):
    for i, (img, d) in enumerate(zip(images, datas)):
        got = img.cpu().numpy() if isinstance(img, torch.Tensor) else np.asarray(img)
        np.testing.assert_array_equal(got, pillow(d), err_msg=f'image {i}')


@pytest.mark.gpu
def test_mixed_batch_and_every_round_cap_equal_pillow():
    datas = corpus() + pillow_only()
    n_pil = len(pillow_only())
    dec = pp.GpuJpegDecoder(len(datas), sum(len(d) for d in datas), 401 * 400)
    for cap in (-1, 0, 1, 2):
        images, routes = dec(datas, max_rounds=cap)
        assert routes == ['gpu'] * len(CORPUS) + ['pillow'] * n_pil
        torch.cuda.synchronize()
        assert_equal_pillow(images, datas)
        st = dec.stats()
        assert (st['gpu'], st['pillow']) == (len(CORPUS), n_pil)
        # the counters equal the restatement's: with cap 0 every subsequence in use is a fallback
        assert (st['sync_rounds'], st['fallbacks']) == expected_stats(datas, cap), (cap, st)
        print(cap, st)
    n_used = sum(len(jr.subsequences(h, *jr.unstuff(d, h['seg']), 1024))
                 for d in datas for r, h in [jr.parse(d)] if r == 'gpu')
    assert expected_stats(datas, 0) == (0, n_used)
    dec.close()


@pytest.mark.gpu
def test_large_photo_equals_pillow():
    datas = [encode(3024, 4032, seed=11, quality=92, subsampling=2),
             encode(3024, 4032, seed=12, quality=80, subsampling=1, restart_marker_rows=2)]
    dec = pp.GpuJpegDecoder(2, sum(len(d) for d in datas), 4032 * 3024)
    for cap in (-1, 1):
        images, routes = dec(datas, max_rounds=cap)
        assert routes == ['gpu', 'gpu']
        assert_equal_pillow(images, datas)
        print(cap, dec.stats())
    dec.close()


@pytest.mark.gpu
def test_malformed_streams_raise_write_nothing_and_the_handle_recovers():
    good = corpus()[:6]
    data = encode(40, 48, quality=90, subsampling=2)
    dec = pp.GpuJpegDecoder(8, 1 << 16, 64 * 64)
    dec._out.fill_(7)
    torch.cuda.synchronize()
    for bad, msg in ((data[:len(data) // 2], 'truncated'), (without(data, b'\xff\xdb'), 'quantisation table missing'),
                     (all_ones_huffman(data), 'bad Huffman table'),
                     (encode(65, 64, quality=90), 'pixel capacity'), (b'not a jpeg', 'SOI')):
        with pytest.raises(RuntimeError, match=msg):
            dec(good[:3] + [bad] + good[3:])
        torch.cuda.synchronize()
        assert bool((dec._out == 7).all()), msg
    with pytest.raises(RuntimeError, match='max_images'):
        dec(good + good)
    images, routes = dec(good)
    assert routes == ['gpu'] * len(good)
    assert_equal_pillow(images, good)
    dec.close()


@pytest.mark.gpu
def test_streams_pillow_decodes_differently_take_the_pillow_route():
    data = encode(24, 32, quality=90, subsampling=0)
    no_dht = without(data, b'\xff\xc4')
    dec = pp.GpuJpegDecoder(2, 1 << 16, 64 * 64)
    images, routes = dec([no_dht, data])
    assert routes == ['pillow', 'gpu']
    assert_equal_pillow(images, [no_dht, data])
    with pytest.raises(OSError):            # routed to Pillow, which refuses it as the reference's loader would
        dec([swapped_scan_order(data)])
    dec.close()


@pytest.mark.gpu
def test_strips_fit_the_decoder_sized_from_their_headers():
    """1 x 20000 and 20000 x 1 strips: many more 8x8 blocks than pixels.  The predictor sizes its decoder from the
    frame headers (`jpeg_footprint`), so they decode, equal to Pillow"""
    import types
    from openpifpaf_b200 import predictor
    datas = [encode(1, 20000, seed=1, quality=90, subsampling=2), encode(20000, 1, seed=2, quality=90, subsampling=0),
             encode(3, 5000, seed=3, quality=90, subsampling=1)]
    for d in datas:
        route, hdr = jr.parse(d)
        assert pp.jpeg_footprint(d) == (hdr['w'] * hdr['h'], hdr['mx'] * hdr['my'] * len(hdr['blocks']))
    host = types.SimpleNamespace(net=types.SimpleNamespace(max_batch=2), device=torch.device('cuda', 0))
    dec = predictor.Predictor._jpeg_decoder(host, datas[:2])
    assert dec.max_blocks == sum(pp.jpeg_footprint(d)[1] for d in datas[:2])
    images, routes = dec(datas[:2])
    assert routes == ['gpu', 'gpu']
    assert_equal_pillow(images, datas[:2])
    dec = predictor.Predictor._jpeg_decoder(host, datas[2:])
    images, _ = dec(datas[2:])
    assert_equal_pillow(images, datas[2:])
    dec.close()


def pose_plan():
    from openpifpaf_b200 import network
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=-2.0)
    for hd in plan['heads']:
        hd['w'] = hd['w'] * np.float32(0.06)
    return plan


@pytest.mark.gpu
def test_jpeg_images_equal_raw_images_on_pillow_arrays(monkeypatch, tmp_path):
    """2 * max_batch + 1 files (paths and bytes, one Pillow-route stream): jpeg_images == raw_images on the arrays
    Pillow decodes, dict for dict with json_data, with and without overlap_decode"""
    from openpifpaf_b200 import constants, decoder, network, predictor
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)     # keep the random-init poses
    S, MB = 161, 2
    shapes = [(120, 161, 2), (161, 100, 1), (300, 200, 0), (90, 250, 2), (161, 161, 2)]
    datas = [encode(h, w, seed=30 + i, quality=90, subsampling=sub) for i, (h, w, sub) in enumerate(shapes)]
    datas[2] = pillow_only()[0]
    files = list(datas)
    for i in (0, 3):
        p = tmp_path / f'{i}.jpg'
        p.write_bytes(datas[i])
        files[i] = str(p)
    arrays = [pillow(d) for d in datas]
    fills = [3, (10, 20, 30), 250, 77, (0, 128, 255)]
    weights = np.linspace(3.0, 1.0, constants.COCO_N_KEYPOINTS)
    for overlap in (False, True):
        pred = predictor.Predictor(network.CompiledNet(pose_plan(), S, S, MB), constants.COCO_N_KEYPOINTS,
                                   constants.COCO_PERSON_SKELETON, overlap_decode=overlap)
        want = pred.raw_images(arrays, fill=fills)
        got = pred.jpeg_images(files, fill=fills)
        assert len(got) == len(files) and sum(d.shape[0] for d, _, _ in want) > 0
        for (d, s, m), (wd, ws, wm) in zip(got, want):
            np.testing.assert_array_equal(d, wd)
            np.testing.assert_array_equal(s, ws)
            for k in ('offset', 'scale', 'valid_area', 'width_height'):
                np.testing.assert_array_equal(m[k], wm[k])
        js = pred.jpeg_images(files, fill=fills, json_data=True, score_weights=weights)
        wjs = pred.raw_images(arrays, fill=fills, json_data=True, score_weights=weights)
        assert [j for j, _ in js] == [j for j, _ in wjs]
        pred.close()


@pytest.mark.gpu
def test_det_predictor_refuses_jpeg_images():
    from openpifpaf_b200 import predictor
    with pytest.raises(RuntimeError, match='not implemented for detection'):
        predictor.DetPredictor.jpeg_images(object.__new__(predictor.DetPredictor), [b''])


# ---------------------------------------------------------------------------------------------------- the reference
REFERENCE_SCRIPT = textwrap.dedent('''
    import sys, warnings
    warnings.filterwarnings('ignore')
    import numpy as np
    import torch
    import torchvision.transforms.functional as TF
    from PIL import Image
    import openpifpaf
    import openpifpaf.transforms.scale as scale_mod
    from openpifpaf.plugins.coco.constants import COCO_PERSON_SCORE_WEIGHTS
    from openpifpaf_b200 import predictor as b200_predictor, synth
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
    with torch.no_grad():                                   # trained-network-like head statistics
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

    shapes = [(900, 1200, 2), (100, 640, 1), (640, 100, 0), (641, 300, 2), (150, 200, 2), (480, 360, 1), (333, 500, 2)]
    paths = []
    for i, (h, w, sub) in enumerate(shapes):
        paths.append(f'img{i}.jpg')
        Image.fromarray(synth.photo_like_image(h, w, 40 + i)).save(paths[-1], quality=90, subsampling=sub,
                                                                    progressive=(i == 4))
    ref = list(predictor.images(paths))
    TF.pad = pad
    assert len(ref) == len(paths) and len(recorded) == len(paths), (len(ref), len(recorded))

    mine = b200_predictor.from_shell(model, 641, 641, B)
    got = mine.jpeg_images(paths, json_data=True, fill=recorded, score_weights=COCO_PERSON_SCORE_WEIGHTS)
    assert mine._jpeg.last_routes == ['gpu'], mine._jpeg.last_routes    # the last chunk: one baseline file
    n = 0
    for i, ((want, _, wmeta), (js, meta)) in enumerate(zip(ref, got)):
        assert js == want, (i, len(js), len(want))
        for k in ('offset', 'scale', 'valid_area', 'width_height'):
            assert np.array_equal(np.asarray(wmeta[k], dtype=np.float64), meta[k]), (i, k, wmeta[k], meta[k])
        n += len(want)
    assert n > 0
    print('JPEG_IMAGES_REF_OK', n, 'poses on', len(paths), 'files, greys', recorded)
''')


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
def test_jpeg_images_equal_reference_predictor_images(tmp_path):
    """the reference's own Predictor.images (batch size 3, long edge 641, PIL decode in its loader, Pillow rescale,
    CenterPad, CifCafB200) on 7 JPEG files == jpeg_images on the same files with the greys its CenterPad drew"""
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', REFERENCE_SCRIPT], capture_output=True, text=True, env=env,
                       cwd=str(tmp_path), timeout=900)
    assert 'JPEG_IMAGES_REF_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout.strip().splitlines()[-1])
