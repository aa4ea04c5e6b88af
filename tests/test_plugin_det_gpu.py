"""GPU: detection models through the reference's own Predictor with this plugin registered (the unmodified reference
package staged in oracle/_ref_pkg, as in tests/test_plugin_gpu.py).  `Multi.batch` must reach `CifDetB200.batch`
for the resnet18-cocodet recipe and for shufflenetv2k16 with the CocoDet upsample-2 head, and its annotations must
equal the reference's own CifDet decoder on the compiled net's fields; a MobileNetV3-small detection model, which the
compiled forward does not implement, must still decode through the reference batch path as before.

Reference call chain exercised (paths relative to the reference's src/openpifpaf/):
  Predictor / Multi.batch              predictor.py:21-153, decoder/multi.py
  CocoDet head metas                   plugins/coco/cocodet.py:43-51
  CifDet (the checker)                 decoder/cifdet.py:15-96
"""
import os
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')

SCRIPT = textwrap.dedent('''
    import json, os, sys, warnings
    warnings.filterwarnings('ignore')
    import numpy as np
    import torch
    import torchvision
    import openpifpaf
    from openpifpaf.network import basenetworks, factory
    torch.ops.openpifpaf.set_quiet(True)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False   # fallback: same fields twice
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED

    # no checkpoint can be downloaded: every backbone from scratch, and torchvision is never asked for weights
    basenetworks.Resnet.pretrained = False
    basenetworks.MobileNetV3.pretrained = False
    factory.BASE_FACTORIES['resnet18'] = lambda: basenetworks.Resnet(
        'resnet18', lambda pretrained: torchvision.models.resnet18(weights=None), 512)
    factory.BASE_FACTORIES['mobilenetv3small'] = lambda: basenetworks.MobileNetV3(
        'mobilenetv3small', lambda pretrained: torchvision.models.mobilenet_v3_small(weights=None), 576)
    openpifpaf.plugins.coco.CocoDet.upsample_stride = 2          # --cocodet-upsample=2
    report = {}
    sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
    from det_models import calibrate_det_head        # the head calibration of the in-process detection tests

    def key(a):
        return (-a.score, a.category_id, tuple(np.round(a.bbox, 3)))

    def compare(got, want, what):
        assert len(got) == len(want), (what, len(got), len(want))
        for a, b in zip(sorted(got, key=key), sorted(want, key=key)):
            assert a.category == b.category and a.category_id == b.category_id, what
            assert abs(a.score - b.score) <= 1e-6, (what, a.score, b.score)
            assert np.abs(np.asarray(a.bbox) - np.asarray(b.bbox)).max() <= 1e-4, what
            assert a.json_data() == b.json_data(), what

    def run(base_name, fast, configure=None):
        torch.manual_seed(0)
        if configure:
            configure()
        openpifpaf.network.Factory.base_name = base_name
        openpifpaf.network.Factory.checkpoint = None
        datamodule = openpifpaf.plugins.coco.CocoDet()
        predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas)
        multi = predictor.processor
        (top,) = [d for d in multi.decoders if d is not None]
        assert type(top).__name__ == 'CifDetB200', type(top).__name__
        calibrate_det_head(predictor.model)
        (meta,) = predictor.model_cpu.head_metas
        ref = openpifpaf.decoder.CifDet([meta])                      # the reference's own decoder: the checker
        calls = []
        orig = type(top).batch
        def spy(self, *a, **k):
            calls.append(1)
            return orig(self, *a, **k)
        type(top).batch = spy
        total = 0
        try:
            for b in (3, 2):                                           # two batch shapes: the compile cache
                images = torch.randn(b, 3, 161, 161, generator=torch.Generator().manual_seed(b))
                got = multi.batch(predictor.model, images, device=predictor.device)
                assert len(got) == b
                if fast:
                    (pred,) = [p for (_, _, p) in top._compiled.values()]
                    (fields,) = pred.fields_batch(images.to(predictor.device))
                    fields = fields.cpu()
                else:
                    with torch.no_grad():
                        (fields,) = predictor.model(images.to(predictor.device))
                    fields = fields.cpu()
                for i in range(b):
                    want = ref([fields[i]])
                    compare(got[i], want, f'{base_name} image {i} of {b}')
                    assert len(want) > 0, (base_name, i)
                    total += len(want)
        finally:
            type(top).batch = orig
        assert len(calls) == 2, calls                                  # Multi.batch reached CifDetB200.batch
        assert bool(top._compiled) == fast
        return total

    def cocodet_recipe():
        basenetworks.Resnet.input_conv2_stride = 2
        basenetworks.Resnet.block5_dilation = 2

    report['resnet18_cocodet'] = run('resnet18', True, cocodet_recipe)
    assert basenetworks.Resnet.pretrained is False
    report['shufflenetv2k16'] = run('shufflenetv2k16', True)
    report['mobilenetv3small_fallback'] = run('mobilenetv3small', False)
    assert basenetworks.MobileNetV3.pretrained is False
    print('PLUGIN_DET_GPU_OK', json.dumps(report))
''')


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
def test_reference_predictor_runs_detection_through_the_plugin(tmp_path):
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', SCRIPT, ROOT], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=900)
    assert 'PLUGIN_DET_GPU_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
