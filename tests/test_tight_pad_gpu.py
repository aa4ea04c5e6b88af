"""GPU: Predictor.raw_images(tight_pad=True) on mixed photo sizes runs every canvas group on one net and equals, image
for image, a net compiled at each canvas size and decoded there; jpeg_images equals raw_images; and where the staged
reference package exists, the reference's own Predictor at batch size 1 (CenterPadTight(16)) gives the same json."""
import io
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from openpifpaf_b200 import constants, decoder, network, predictor, synth
from openpifpaf_b200 import preprocess as pp

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')
SHAPES = [(240, 320), (320, 240), (161, 161), (200, 300), (240, 320), (96, 321), (300, 200), (150, 100), (240, 320)]


def pose_plan():
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=-2.0)
    for hd in plan['heads']:
        hd['w'] = hd['w'] * np.float32(0.06)
    return plan


def make_predictor(plan, h, w, max_batch):
    return predictor.Predictor(network.CompiledNet(plan, h, w, max_batch), constants.COCO_N_KEYPOINTS,
                               constants.COCO_PERSON_SKELETON)


@pytest.mark.parametrize('long_edge,backend', [(321, 'pillow'), (None, 'pillow'), (257, 'scipy'), (321, 'opencv')])
def test_tight_pad_equals_a_net_compiled_at_each_canvas(monkeypatch, long_edge, backend):
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)     # keep the random-init poses
    plan = pose_plan()
    images = [synth.photo_like_image(h, w, seed=i) for i, (h, w) in enumerate(SHAPES)]
    kw = dict(fast_rescaling=backend != 'scipy', opencv_rescaling=backend == 'opencv')
    pred = make_predictor(plan, 321, 321, 2)
    got = pred.raw_images(images, tight_pad=True, long_edge=long_edge, **kw)
    assert pred.net.input_size == (321, 321)              # restored
    groups = predictor.tight_pad_groups([(w, h) for h, w in SHAPES], long_edge, 2, (321, 321))
    assert len({c for c, _ in groups}) >= 3
    n = 0
    for canvas, idx in groups:
        exact = make_predictor(plan, *canvas, 2)
        want = exact.raw_images([images[i] for i in idx], tight_pad=True, long_edge=long_edge, **kw)
        assert exact.net.input_size == canvas
        for i, (wd, ws, wmeta) in zip(idx, want):
            data, scales, meta = got[i]
            np.testing.assert_array_equal(data, wd, err_msg=f'image {i}')
            np.testing.assert_array_equal(scales, ws, err_msg=f'image {i}')
            for k in ('offset', 'scale', 'valid_area', 'width_height'):
                assert np.array_equal(meta[k], wmeta[k]), (i, k)
            n += len(wd)
        exact.close()
    assert n > 0
    # the capacity net still runs its own size afterwards, and a canvas above it is refused up front
    with pytest.raises(RuntimeError, match='above the net'):
        pred.raw_images([images[0], synth.photo_like_image(400, 300, seed=9)], tight_pad=True, long_edge=400)
    assert pred.net.input_size == (321, 321)
    pred.close()


def test_jpeg_images_equal_raw_images(monkeypatch):
    PIL = pytest.importorskip('PIL.Image')
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)
    blobs, images = [], []
    for i, (h, w) in enumerate(SHAPES[:6]):
        buf = io.BytesIO()
        PIL.fromarray(synth.photo_like_image(h, w, seed=20 + i)).save(buf, format='JPEG', quality=90)
        blobs.append(buf.getvalue())
        images.append(np.asarray(PIL.open(io.BytesIO(blobs[-1])).convert('RGB')))
    pred = make_predictor(pose_plan(), 321, 321, 2)
    for long_edge in (321, None):
        want = pred.raw_images(images, tight_pad=True, long_edge=long_edge, json_data=True)
        got = pred.jpeg_images(blobs, tight_pad=True, long_edge=long_edge, json_data=True)
        assert [j for j, _ in got] == [j for j, _ in want]
    pred.close()


REFERENCE_SCRIPT = textwrap.dedent('''
    import sys, warnings
    warnings.filterwarnings('ignore')
    import numpy as np
    import torch
    import openpifpaf
    import openpifpaf.transforms.scale as scale_mod
    from openpifpaf.plugins.coco.constants import COCO_PERSON_SCORE_WEIGHTS
    from openpifpaf_b200 import predictor as b200_predictor
    torch.ops.openpifpaf.set_quiet(True)
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED
    scale_mod.cv2 = None                                    # the Pillow path of RescaleAbsolute (transforms/scale.py:56-59)
    long_edge = None if sys.argv[1] == 'none' else int(sys.argv[1])
    openpifpaf.Predictor.batch_size = 1                     # the default: CenterPadTight(16) (predictor.py:94-95)
    openpifpaf.Predictor.long_edge = long_edge
    openpifpaf.Predictor.loader_workers = 0
    torch.manual_seed(0)
    openpifpaf.network.Factory.base_name = 'shufflenetv2k16'
    openpifpaf.network.Factory.checkpoint = None
    datamodule = openpifpaf.plugins.coco.CocoKp()
    predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas, json_data=True)
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
    rng = np.random.default_rng(5)
    shapes = [(480, 640), (640, 480), (100, 640), (333, 500), (150, 200), (480, 360), (480, 640)]
    if long_edge is None:
        # native size: half the photos' sides keeps the poses of noise images under the decoder's 512 per image
        shapes = [(h // 2, w // 2) for h, w in shapes]
    raw = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for (h, w) in shapes]
    ref = list(predictor.numpy_images(raw))
    mine = b200_predictor.from_shell(model, 641, 641, 3)
    got = mine.raw_images(raw, json_data=True, tight_pad=True, long_edge=long_edge,
                          score_weights=COCO_PERSON_SCORE_WEIGHTS)
    n = 0
    for i, ((want, _, wmeta), (js, meta)) in enumerate(zip(ref, got)):
        assert js == want, (i, len(js), len(want))
        for k in ('offset', 'scale', 'valid_area', 'width_height'):
            assert np.array_equal(np.asarray(wmeta[k], dtype=np.float64), meta[k]), (i, k, wmeta[k], meta[k])
        n += len(want)
    assert n > 0
    print('TIGHT_PAD_REF_OK', n, 'poses on', len(raw), 'images')
''')


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
@pytest.mark.parametrize('long_edge', ['none', '641'])
def test_tight_pad_equals_reference_predictor_at_batch_size_1(tmp_path, long_edge):
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', REFERENCE_SCRIPT, long_edge], capture_output=True, text=True, env=env,
                       cwd=str(tmp_path), timeout=900)
    assert 'TIGHT_PAD_REF_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout.strip().splitlines()[-1])
