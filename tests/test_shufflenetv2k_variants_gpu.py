"""GPU: ShuffleNetV2K with the structural options of tests/test_shufflenetv2k_variants.py in the compiled forward.
The dilated depthwise conv (the dilation-2 mode of the TMA kernel, and the generic kernel for other dilations and
shapes) against float64 with the sentinels, bounds and column windows of tests/test_kernels_gpu.py, bit for bit against
each other and across launch schedules; the refusals of pifpaf_net_dwconv_dilated; every variant op by op against the
float64 reference of what the GPU fed each op and against fp32 PyTorch, in both activation layouts; shufflenetv2k16 with
stage-4 dilation 2 at 641 px; Predictor on a dilated model against the decoder on the compiled fields; and the
reference's own Predictor with --shufflenetv2k-stage4-dilation 2 through the plugin."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import kernel_refs as kr
import mobilenetv2_models as mm
import shufflenetv2k_models as sm
from openpifpaf_b200 import _lib, decoder, network, predictor
from test_kernels_gpu import Case, Check, check_ops_teacher_forced, n_sm, pad8, pad16, ptr

pytestmark = pytest.mark.gpu

FIELD_TOL_REL = 3e-2        # tests/test_network_gpu.py


# (H, W, channels, kernel, dilation, pad, in_off, out_off, relu, batch, max_batch)
TMA_CASES = [                                       # 5x5, dilation 2, stride 1: DW_K5_S1_D2
    (1, 1, 16, 5, 2, 4, 0, 0, 1, 1, 2),             # one pixel: every tap but the centre in the padding
    (5, 7, 48, 5, 2, 4, 0, 0, 0, 2, 3),             # smaller than one 8 x 16 tile, 48 channels
    (8, 16, 64, 5, 2, 4, 0, 0, 1, 1, 2),            # exactly one tile
    (13, 11, 96, 5, 2, 4, 16, 0, 1, 2, 3),          # column window of the input, partial tiles
    (17, 19, 40, 5, 2, 4, 0, 16, 0, 2, 3),          # column window of the output, 40 channels
    (19, 23, 72, 5, 2, 0, 8, 8, 1, 1, 2),           # pad 0: the output shrinks by 8
    (41, 43, 176, 5, 2, 4, 0, 0, 1, 2, 3),          # 176 = 2 x 64 + 48
    (81, 81, 352, 5, 2, 4, 0, 0, 0, 1, 2),          # stage 4 of shufflenetv2k16 at 641 px (branch2)
    (81, 81, 704, 5, 2, 4, 0, 0, 0, 1, 1),          # its block-0 branch1
]
GENERIC_CASES = [                                   # the generic kernel
    (9, 10, 40, 5, 3, 6, 0, 0, 1, 2, 3),            # dilation 3
    (23, 21, 96, 5, 3, 6, 8, 16, 0, 1, 2),
    (12, 13, 72, 3, 2, 2, 0, 0, 1, 2, 3),           # 3x3, dilation 2
    (11, 13, 24, 5, 2, 4, 0, 0, 2, 2, 3),           # 5x5, dilation 2 with ReLU6
]


def dw_id(c):
    return 'H%dW%d-C%d-k%dd%dp%d-in%d-out%d-act%d-B%dof%d' % c


def dwd_case(H, W, C, k, d, pad, in_off, out_off, relu, batch, mb, seed=0):
    Ho, Wo = kr.out_hw(H, W, (k - 1) * d + 1, 1, pad)
    case = Case(mb, [(H, W, pad16(in_off + pad8(C) + 8)), (Ho, Wo, pad16(out_off + pad8(C) + 16))], inputs={0},
                seed=seed)
    rng = np.random.default_rng(seed + 1)
    w = (2 * rng.standard_normal((C, k, k)) / k).astype(np.float32)        # f32 weights: not rounded to bf16
    b = rng.uniform(-3.0, 9.0, C).astype(np.float32)

    def emit(L, net):
        _lib.check(L.pifpaf_net_dwconv_dilated(net, 0, in_off, C, k, 1, pad, ptr(w), ptr(b), relu, 1, out_off, d))

    x = case.data[0][:batch, ..., in_off:in_off + C]
    ref, mag = kr.epilogue(*kr.conv_ref(x, w.reshape(C, 1, k, k), b, 1, pad, groups=C, dilation=d), relu)
    chk = Check('dwconv k%d dilated' % k, batch)
    chk.own(1, out_off, out_off + pad8(C))
    chk.compare(1, out_off, ref, kr.bf16_bound(ref, mag, k * k))
    return case, emit, chk


@pytest.mark.parametrize('c', TMA_CASES, ids=dw_id)
def test_dilated_dwconv_tma_matches_float64_and_generic_bitwise(c):
    case, emit, chk = dwd_case(*c)
    taps, _ = case.run(emit, c[9])
    chk.kind += ' tma'
    print(dw_id(c), '%.3f' % chk.verify(taps, dw_id(c)))
    generic, _ = case.run(emit, c[9], impl=1)           # gemm_impl = 1: k_dwconv
    np.testing.assert_array_equal(taps[1], generic[1])


@pytest.mark.parametrize('c', GENERIC_CASES, ids=dw_id)
def test_dilated_dwconv_generic_matches_float64(c):
    case, emit, chk = dwd_case(*c)
    for impl in (0, 1):
        taps, _ = case.run(emit, c[9], impl=impl)
        print(dw_id(c), impl, '%.3f' % chk.verify(taps, f'{dw_id(c)} impl {impl}'))


@pytest.mark.parametrize('c', [TMA_CASES[6], TMA_CASES[7], GENERIC_CASES[1]], ids=dw_id)
def test_dilated_dwconv_schedules_are_bitwise_invariant(c, monkeypatch):
    """the persistent grid at SM limits 1 / 7 / n_sm - 4 and without programmatic dependent launch"""
    case, emit, _ = dwd_case(*c)
    want, _ = case.run(emit, c[9])
    for lim in (1, 7, n_sm() - 4):
        got, _ = case.run(emit, c[9], sm_limit=lim)
        assert np.array_equal(got[1], want[1]), lim
    monkeypatch.setenv('PIFPAF_PDL', '0')
    got, _ = case.run(emit, c[9])
    assert np.array_equal(got[1], want[1])


def test_dilated_dwconv_refusals():
    L = _lib.lib()
    net = ctypes.c_void_p()
    _lib.check(L.pifpaf_net_create(ctypes.byref(net), 0, 1))
    try:
        tid = ctypes.c_int32()
        for h in (17, 9, 17):
            _lib.check(L.pifpaf_net_tensor(net, h, h, 64, ctypes.byref(tid)))
        w = np.zeros((64, 25), dtype=np.float32)
        b = np.zeros(64, dtype=np.float32)
        assert L.pifpaf_net_dwconv_dilated(net, 0, 0, 64, 5, 2, 4, ptr(w), ptr(b), 0, 1, 0, 2) == _lib.E_BADARG
        assert b'stride 1' in L.pifpaf_last_error()
        assert L.pifpaf_net_dwconv_dilated(net, 0, 0, 64, 5, 1, 2, ptr(w), ptr(b), 0, 2, 0, 0) == _lib.E_BADARG
        assert b'dilation' in L.pifpaf_last_error()
        assert L.pifpaf_net_num_ops(net) == 0
        _lib.check(L.pifpaf_net_dwconv_dilated(net, 0, 0, 64, 5, 1, 4, ptr(w), ptr(b), 0, 2, 0, 2))
        assert L.pifpaf_net_num_ops(net) == 1
    finally:
        L.pifpaf_net_destroy(net)


# ---------------------------------------------------------------------------------------------------- networks
def k16_variant_shell(variant, seed):
    return sm.make_pose_shell(variant, 'shufflenetv2k16', seed=seed)


@pytest.mark.parametrize('layout', ['bins', 'shuffle'])
@pytest.mark.parametrize('variant', list(sm.VARIANTS))
def test_variant_teacher_forced_and_against_fp32(variant, layout):
    shell = k16_variant_shell(variant, seed=4)
    plan = network.plan_from_shell(shell)
    H, W, B = 129, 97, 2
    _, ops, _ = network.build_ops(plan, H, W, layout=layout)
    net = network.CompiledNet(plan, H, W, B, layout=layout)
    images = np.random.default_rng(9).standard_normal((B, 3, H, W)).astype(np.float32)
    x = torch.from_numpy(images).cuda()
    worst, got = check_ops_teacher_forced(net, ops, images, 'shufflenetv2k variants', f'{variant} {layout}')
    print(variant, layout, {k: round(v, 3) for k, v in worst.items()})
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        want = shell.cuda()(x)
    for g, wt in zip(got, want):
        assert g.shape == wt.shape
        err = (g - wt).abs()
        assert float(err.max()) < FIELD_TOL_REL * float(wt.std()) + 1e-3
        assert float(err.mean()) < 1e-2 * float(wt.std())
    net.close()


@pytest.mark.parametrize('variant', ['conv2', 'conv2_out48'])
def test_input_conv2_fused_and_two_kernel_schedules_are_bitwise_equal(variant, monkeypatch):
    """24 channels after the second input conv: the stage-2 entry pair runs as one k_pw_dw launch; 48 channels: as
    two launches.  Either way PIFPAF_FUSE_PW_DW=0 gives the same fields."""
    plan = network.plan_from_shell(k16_variant_shell(variant, seed=5))
    x = torch.randn(2, 3, 161, 161, generator=torch.Generator().manual_seed(3)).cuda()
    fields, kinds = {}, {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('PIFPAF_FUSE_PW_DW', fuse)
        net = network.CompiledNet(plan, 161, 161, 2)
        fields[fuse] = [t.clone() for t in net.forward(x)]
        kinds[fuse] = net.forward_timed(x)[1]
        net.close()
    for a, b in zip(fields['1'], fields['0']):
        assert torch.equal(a, b)
    # forward_timed reports the elided 1x1 op and the k_pw_dw launch as kind 3
    assert int((kinds['1'] == 3).sum()) == (2 if variant == 'conv2' else 0)
    assert int((kinds['0'] == 3).sum()) == 0


def test_k16_dilated_at_641_matches_fp32():
    """shufflenetv2k16 with stage-4 dilation 2 at the benchmark's size: 81 x 81 fields"""
    shell = k16_variant_shell('dil2', seed=6)
    net = network.CompiledNet(network.plan_from_shell(shell), 641, 641, 2)
    x = torch.randn(2, 3, 641, 641, generator=torch.Generator().manual_seed(2)).cuda()
    got = [t.clone() for t in net.forward(x)]
    net.close()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        want = shell.cuda()(x)
    assert tuple(got[0].shape) == (2, 17, 5, 81, 81) and tuple(got[1].shape) == (2, 19, 8, 81, 81)
    for g, wt in zip(got, want):
        assert g.shape == wt.shape
        err = (g - wt).abs()
        assert float(err.max()) < FIELD_TOL_REL * float(wt.std()) + 1e-3
        assert float(err.mean()) < 1e-2 * float(wt.std())


def test_predictor_on_a_dilated_model_equals_cifcaf_on_the_compiled_fields():
    shell = mm.calibrate_pose_heads(k16_variant_shell('dil2_conv5stage', seed=5))
    pred = predictor.from_shell(shell, 161, 161, 4)
    assert pred.net.heads[0]['stride'] == 8 and (pred.net.heads[0]['h'], pred.net.heads[0]['w']) == (21, 21)
    images = torch.randn(4, 3, 161, 161, generator=torch.Generator().manual_seed(3)).pin_memory()
    sk = torch.tensor(shell.head_nets[1].meta.skeleton, dtype=torch.int64) - 1
    total = 0
    for b in (4, 3):
        res = pred.batch(images[:b])
        cif, caf = pred.fields_batch(images[:b].cuda())
        want = decoder.CifCaf(17, sk).decode_batch(cif, 8, caf, 8)
        assert len(res) == len(want) == b
        for (a, i), (wa, wi) in zip(res, want):
            assert torch.equal(a, wa) and torch.equal(i, wi)
            total += int(a.shape[0])
    print('annotations', total)
    pred.close()


# ---------------------------------------------------------------------------------------------------- plugin
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')

SCRIPT = textwrap.dedent('''
    import json, os, sys, warnings
    warnings.filterwarnings('ignore')
    import numpy as np
    import torch
    import openpifpaf
    from openpifpaf.network import basenetworks
    torch.ops.openpifpaf.set_quiet(True)
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED
    basenetworks.ShuffleNetV2K.stage4_dilation = 2      # as configure() sets it for --shufflenetv2k-stage4-dilation 2
    sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
    import mobilenetv2_models

    torch.manual_seed(0)
    openpifpaf.network.Factory.base_name = 'shufflenetv2k16'
    openpifpaf.network.Factory.checkpoint = None
    datamodule = openpifpaf.plugins.coco.CocoKp()
    predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas)
    assert predictor.model_cpu.base_net.stride == 8
    multi = predictor.processor
    (top,) = [d for d in multi.decoders if d is not None]
    assert type(top).__name__ == 'CifCafB200', type(top).__name__
    mobilenetv2_models.calibrate_pose_heads(predictor.model)
    ref = openpifpaf.decoder.CifCaf(predictor.model_cpu.head_metas[:1], predictor.model_cpu.head_metas[1:2])
    calls = []
    orig = type(top).batch
    def spy(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)
    type(top).batch = spy
    total = 0
    try:
        images = torch.randn(3, 3, 161, 161, generator=torch.Generator().manual_seed(3))
        got = multi.batch(predictor.model, images, device=predictor.device)
        (pred,) = [p for (_, _, p) in top._compiled.values()]
        assert pred.net.heads[0]['stride'] == 8
        cif, caf = [f.cpu() for f in pred.fields_batch(images.to(predictor.device))]
        for i in range(3):
            want = ref([cif[i], caf[i]])
            assert len(got[i]) == len(want), (i, len(got[i]), len(want))
            for a, b in zip(sorted(got[i], key=lambda a: -a.score), sorted(want, key=lambda a: -a.score)):
                assert abs(a.score - b.score) <= 1e-5
                assert np.abs(a.data[:, :2] - b.data[:, :2]).max() <= 1e-4
                assert np.abs(a.data[:, 2] - b.data[:, 2]).max() <= 1e-5
            total += len(want)
    finally:
        type(top).batch = orig
    assert calls and top._compiled
    print('PLUGIN_SHUFFLENETV2K_DILATED_OK', json.dumps({'annotations': total}))
''')


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
def test_reference_predictor_runs_dilated_shufflenetv2k_through_the_plugin(tmp_path):
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', SCRIPT, ROOT], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=900)
    assert 'PLUGIN_SHUFFLENETV2K_DILATED_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
