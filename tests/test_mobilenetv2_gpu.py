"""GPU: MobileNetV2 in the compiled forward.  The ReLU6 activation code on every kernel that applies an activation
(stem, the per-lane k_gemm_wg epilogue with and without a residual, the implicit-GEMM conv, the SIMT debug GEMM, the TMA and
generic depthwise kernels) against float64 with values on both sides of 0 and 6; the 3x3 mode of the TMA depthwise
kernel against float64 and bit for bit against the generic kernel (gemm_impl=1); refusals of code 2 where it is not
implemented; a seeded MobileNetV2 with CocoKp heads op by op against the float64 reference of what the GPU fed each op
and against fp32 PyTorch; Predictor / DetPredictor from the Shell against the decoders on the compiled fields; and the
reference's own Predictor with base_name='mobilenetv2' through the plugin.  Sentinels, bounds and column windows are
those of tests/test_kernels_gpu.py."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import det_models
import kernel_refs as kr
import mobilenetv2_models as mm
from openpifpaf_b200 import _lib, decoder, network, predictor
from test_kernels_gpu import Case, Check, n_sm, pad8, pad16, ptr, record

pytestmark = pytest.mark.gpu

FIELD_TOL_REL = 3e-2        # tests/test_network_gpu.py
RELU6 = network.ACT_RELU6


def epilogue(y, mag, code, res=None):
    """+ residual, then the activation of code (0 none, 1 ReLU, 2 ReLU6); both are 1-Lipschitz, the bound carries over"""
    y, mag = kr.epilogue(y, mag, code >= 1, res)
    return (np.minimum(y, 6.0) if code == 2 else y), mag


def straddling_bias(rng, n):
    """biases that put the pre-activations on both sides of 0 and of 6"""
    return rng.uniform(-3.0, 9.0, n).astype(np.float32)


def assert_straddles(ref):
    assert (ref == 0).any() and (ref == 6).any() and ((ref > 0) & (ref < 6)).any()


# ---------------------------------------------------------------------------------------------------- stem
@pytest.mark.parametrize('u8', [False, True], ids=['f32', 'u8'])
def test_input_conv_relu6(u8):
    H, W, C, batch, mb = 33, 31, 32, 2, 3
    Ho, Wo = kr.out_hw(H, W, 3, 2, 1)
    case = Case(mb, [(Ho, Wo, pad16(C + 8))], inputs=set())
    rng = np.random.default_rng(4)
    w = (rng.standard_normal((C, 3, 3, 3)) / 3).astype(np.float32)
    b = straddling_bias(rng, C)
    if u8:
        raw = rng.integers(0, 256, (batch, H, W, 3), dtype=np.uint8)
        x = kr.normalise_u8(raw, network.CompiledNet.IMAGE_MEAN, network.CompiledNet.IMAGE_STD)
        kw = {'u8': raw}
    else:
        images = (2 * rng.standard_normal((batch, 3, H, W))).astype(np.float32)
        x, kw = images.transpose(0, 2, 3, 1), {'images': images}

    def emit(L, net):
        _lib.check(L.pifpaf_net_input_conv(net, H, W, 3, 2, 1, C, ptr(w), ptr(b), RELU6, 0))

    ref, mag = epilogue(*kr.conv_ref(x, w, b, 2, 1), RELU6)
    assert_straddles(ref)
    chk = Check('relu6 input_conv', batch)
    chk.own(0, 0, pad8(C))
    chk.compare(0, 0, ref, kr.bf16_bound(ref, mag, 27))
    taps, _ = case.run(emit, batch, **kw)
    chk.verify(taps)


# ---------------------------------------------------------------------------------------------------- GEMM / conv
# (H, W, c_in, kernel, stride, N, in_off, residual col (None: no residual), out_off, batch, max_batch)
CONV6_CASES = [
    (19, 23, 16, 1, 1, 96, 0, None, 0, 2, 3),        # expand: K = 16 (ReLU6 GEMMs take the per-lane epilogue)
    (21, 21, 160, 1, 1, 960, 0, None, 16, 1, 2),     # wide N, column window
    (41, 41, 96, 1, 1, 24, 8, None, 0, 2, 3),        # N = 24: the per-lane tail of a 32-wide tile
    (17, 19, 144, 1, 1, 24, 0, 8, 0, 2, 3),          # projection with residual: the per-lane epilogue
    (21, 21, 960, 1, 1, 160, 0, 0, 16, 2, 2),
    (17, 19, 72, 3, 2, 80, 8, None, 16, 2, 3),       # implicit-GEMM conv
    (13, 15, 64, 3, 1, 48, 0, 8, 0, 2, 2),
]


def conv6_id(c):
    return 'H%dW%d-cin%d-k%ds%d-N%d-in%d-res%s-out%d-B%dof%d' % c


def conv6_case(H, W, c_in, k, stride, N, in_off, res_col, out_off, batch, mb, seed=0):
    pad = (k - 1) // 2
    Ho, Wo = kr.out_hw(H, W, k, stride, pad)
    tensors = [(H, W, pad16(in_off + c_in + 8)), (Ho, Wo, pad16(out_off + pad8(N) + 16))]
    inputs = {0}
    if res_col is not None:
        tensors.append((Ho, Wo, pad16(res_col + N + 8)))
        inputs.add(2)
    case = Case(mb, tensors, inputs=inputs, seed=seed)
    rng = np.random.default_rng(seed + 3)
    w = kr.random_bf16(rng, (N, c_in, k, k), 1 / np.sqrt(c_in * k * k))
    b = straddling_bias(rng, N)

    def emit(L, net):
        _lib.check(L.pifpaf_net_conv(net, 0, in_off, c_in, k, stride, pad, N, ptr(w), ptr(b), RELU6, 1, out_off,
                                     -1 if res_col is None else 2, 0 if res_col is None else res_col))

    ref, mag = kr.conv_ref(case.data[0][:batch, ..., in_off:in_off + c_in], w, b, stride, pad)
    res = None if res_col is None else case.data[2][:batch, ..., res_col:res_col + N]
    ref, mag = epilogue(ref, mag, RELU6, res)
    assert_straddles(ref)
    chk = Check('relu6 conv k%d%s' % (k, '' if res_col is None else ' residual'), batch)
    chk.own(1, out_off, out_off + pad8(N))
    chk.compare(1, out_off, ref, kr.bf16_bound(ref, mag, c_in * k * k))
    return case, emit, chk


@pytest.mark.parametrize('impl', [0, 1], ids=['wgmma', 'simt'])
@pytest.mark.parametrize('c', CONV6_CASES, ids=conv6_id)
def test_conv_relu6_matches_float64(c, impl, monkeypatch):
    case, emit, chk = conv6_case(*c)
    taps, _ = case.run(emit, c[9], impl=impl)
    chk.kind += ' simt' if impl else ''
    print(conv6_id(c), impl, '%.3f' % chk.verify(taps, conv6_id(c)))
    if impl == 0 and c[3] == 1 and c[7] is None:
        # PIFPAF_GEMM_TMA_STORE=0 gives the same bits (ReLU6 GEMMs never take the TMA-store epilogue)
        monkeypatch.setenv('PIFPAF_GEMM_TMA_STORE', '0')
        lane, _ = case.run(emit, c[9])
        np.testing.assert_array_equal(lane[1], taps[1])


def test_conv1x1_plain_relu6():
    """pifpaf_net_conv1x1 (plain output) with code 2, and the codes it refuses"""
    h, w, K, N, batch, mb = 23, 29, 96, 144, 2, 3
    case = Case(mb, [(h, w, pad16(K + 8)), (h, w, pad16(N) + 16), (h, w, pad16(N))], inputs={0, 2})
    rng = np.random.default_rng(8)
    wt = kr.random_bf16(rng, (N, K), 1 / np.sqrt(K))
    b = straddling_bias(rng, N)

    def emit(L, net):
        _lib.check(L.pifpaf_net_conv1x1(net, 0, 0, K, N, ptr(wt), ptr(b), RELU6, 1, 0, -1, 0))
        assert L.pifpaf_net_conv1x1(net, 0, 0, K, N, ptr(wt), ptr(b), RELU6, 1, 0, 2, 0) == _lib.E_BADARG
        assert L.pifpaf_net_conv1x1(net, 0, 0, K, N, ptr(wt), ptr(b), 3, 1, 0, -1, 0) == _lib.E_BADARG
        assert L.pifpaf_net_num_ops(net) == 1

    ref, mag = epilogue(*kr.conv_ref(case.data[0][:batch, ..., :K], wt[:, :, None, None], b, 1, 0), RELU6)
    assert_straddles(ref)
    chk = Check('relu6 gemm plain', batch)
    chk.own(1, 0, N)
    chk.compare(1, 0, ref, kr.bf16_bound(ref, mag, K))
    for impl in (0, 1):
        taps, _ = case.run(emit, batch, impl=impl)
        chk.verify(taps, f'impl {impl}')


def test_relu6_is_refused_where_it_is_not_implemented():
    L = _lib.lib()
    net = ctypes.c_void_p()
    _lib.check(L.pifpaf_net_create(ctypes.byref(net), 0, 1))
    try:
        tid = ctypes.c_int32()
        for _ in range(3):
            _lib.check(L.pifpaf_net_tensor(net, 9, 9, 64, ctypes.byref(tid)))
        w = np.zeros((64, 64), dtype=np.float32)
        dw = np.zeros((64, 25), dtype=np.float32)
        b = np.zeros(64, dtype=np.float32)
        one = [ctypes.byref(ctypes.c_int32(v)) for v in (0, 64, 1, 0)]
        assert L.pifpaf_net_conv1x1_scatter(net, 0, 0, 64, 64, ptr(w), ptr(b), RELU6, 1, *one) == _lib.E_BADARG
        for dw_relu, relu in ((RELU6, 1), (0, RELU6)):
            assert L.pifpaf_net_dw_conv1x1_scatter(net, 0, 0, 64, 5, 1, 2, ptr(dw), ptr(b), dw_relu, 64, ptr(w), ptr(b),
                                                   relu, 1, *one) == _lib.E_BADARG
        assert L.pifpaf_net_dwconv(net, 0, 0, 64, 3, 1, 1, ptr(dw), ptr(b), 3, 1, 0) == _lib.E_BADARG
        assert L.pifpaf_net_dwconv(net, 0, 0, 64, 3, 1, 1, ptr(dw), ptr(b), -1, 1, 0) == _lib.E_BADARG
        assert L.pifpaf_net_input_conv(net, 17, 17, 3, 2, 1, 16, ptr(w), ptr(b), 3, 0) == _lib.E_BADARG
        assert b'activation' in L.pifpaf_last_error()
        assert L.pifpaf_net_num_ops(net) == 0
    finally:
        L.pifpaf_net_destroy(net)


# ---------------------------------------------------------------------------------------------------- depthwise
# (H, W, channels, kernel, stride, pad, in_off, out_off, relu, batch, max_batch)
DW3_CASES = [
    (1, 1, 16, 3, 1, 1, 0, 0, 2, 1, 2),
    (8, 16, 16, 3, 1, 1, 0, 0, 2, 2, 3),            # exactly one 8 x 16 tile
    (9, 17, 32, 3, 2, 1, 16, 0, 2, 1, 2),           # column window of the input
    (13, 11, 96, 3, 1, 1, 0, 16, 2, 3, 4),          # column window of the output, partial tiles
    (37, 23, 144, 3, 2, 1, 0, 0, 2, 2, 3),          # 144 = 2 x 64 + 16
    (21, 21, 960, 3, 1, 1, 0, 0, 2, 2, 2),          # 15 channel blocks
    (41, 41, 960, 3, 2, 1, 8, 8, 2, 1, 2),
    (12, 9, 72, 3, 2, 0, 0, 0, 1, 2, 3),            # pad 0, ReLU
    (17, 19, 40, 3, 1, 1, 0, 0, 0, 1, 2),           # no activation
    (161, 161, 144, 3, 1, 1, 0, 0, 2, 2, 3),        # the slot ring wraps many times
    (321, 321, 96, 3, 2, 1, 0, 0, 2, 1, 2),         # stage-2 entry of a 641 px image
    (161, 161, 144, 3, 2, 1, 0, 0, 2, 3, 4),
]
DW6_OTHER = [                                       # ReLU6 on the other depthwise kernels
    (19, 23, 72, 5, 1, 2, 0, 8, 2, 2, 3),           # 5x5 with code 2: k_dwconv5
    (19, 23, 72, 5, 2, 2, 8, 0, 2, 2, 3),
    (17, 19, 44, 7, 1, 3, 0, 0, 2, 2, 3),           # k_dwconv
]


def dw_id(c):
    return 'H%dW%d-C%d-k%ds%dp%d-in%d-out%d-act%d-B%dof%d' % c


def dw_case(H, W, C, k, stride, pad, in_off, out_off, relu, batch, mb, seed=0):
    Ho, Wo = kr.out_hw(H, W, k, stride, pad)
    case = Case(mb, [(H, W, pad16(in_off + pad8(C) + 8)), (Ho, Wo, pad16(out_off + pad8(C) + 16))], inputs={0},
                seed=seed)
    rng = np.random.default_rng(seed + 1)
    w = (2 * rng.standard_normal((C, k, k)) / k).astype(np.float32)        # f32 weights: not rounded to bf16
    b = straddling_bias(rng, C)

    def emit(L, net):
        _lib.check(L.pifpaf_net_dwconv(net, 0, in_off, C, k, stride, pad, ptr(w), ptr(b), relu, 1, out_off))

    x = case.data[0][:batch, ..., in_off:in_off + C]
    ref, mag = epilogue(*kr.conv_ref(x, w.reshape(C, 1, k, k), b, stride, pad, groups=C), relu)
    if relu == 2 and ref.size > 1000:
        assert_straddles(ref)
    chk = Check('relu6 dwconv k%d s%d' % (k, stride) if relu == 2 else 'dwconv k%d s%d' % (k, stride), batch)
    chk.own(1, out_off, out_off + pad8(C))
    chk.compare(1, out_off, ref, kr.bf16_bound(ref, mag, k * k))
    return case, emit, chk


@pytest.mark.parametrize('c', DW3_CASES, ids=dw_id)
def test_dwconv3_tma_matches_float64_and_generic_bitwise(c):
    case, emit, chk = dw_case(*c)
    taps, _ = case.run(emit, c[9])
    chk.kind += ' tma'
    print(dw_id(c), '%.3f' % chk.verify(taps, dw_id(c)))
    generic, _ = case.run(emit, c[9], impl=1)
    np.testing.assert_array_equal(taps[1], generic[1])


@pytest.mark.parametrize('c', DW6_OTHER, ids=dw_id)
def test_dwconv_relu6_other_kernels(c):
    case, emit, chk = dw_case(*c)
    for impl in (0, 1):
        taps, _ = case.run(emit, c[9], impl=impl)
        chk.verify(taps, f'{dw_id(c)} impl {impl}')


@pytest.mark.parametrize('c', [DW3_CASES[4], DW3_CASES[9]], ids=dw_id)
def test_dwconv3_tma_schedules_are_bitwise_invariant(c, monkeypatch):
    case, emit, _ = dw_case(*c)
    want, _ = case.run(emit, c[9])
    for lim in (1, 7, n_sm() - 4):
        got, _ = case.run(emit, c[9], sm_limit=lim)
        assert np.array_equal(got[1], want[1]), lim
    monkeypatch.setenv('PIFPAF_PDL', '0')
    got, _ = case.run(emit, c[9])
    assert np.array_equal(got[1], want[1])


# ---------------------------------------------------------------------------------------------------- network
def op_check(o, taps, heads, images, batch):
    """float64 reference of one MobileNetV2 op from the tensors the GPU fed it -> (kind, worst err / bound)"""
    kind = o['kind']

    def a_in(t, off, n):
        return taps[t][:batch, ..., off:off + n]

    if kind == 'heads':
        refs = kr.heads_ref(a_in(o['in'], 0, o['k_cols']), kr.bf16_round(o['w']), o['b'], o['n_fields'], o['n_comp'],
                            o['ops'])
        return 'heads', max(kr.worst_ratio(hb[:batch], r, bd) for hb, (r, bd) in zip(heads, refs))
    if kind == 'input_conv':
        ref, mag = epilogue(*kr.conv_ref(images[:batch].transpose(0, 2, 3, 1), o['w'], o['b'], o['stride'], o['pad']),
                            o['relu'])
        return kind, kr.worst_ratio(taps[o['out']][:batch, ..., :o['c_out']], ref, kr.bf16_bound(ref, mag, 27))
    if kind == 'dwconv':
        C, k = o['channels'], o['kernel']
        ref, mag = epilogue(*kr.conv_ref(a_in(o['in'], o['in_off'], C), o['w'].reshape(C, 1, k, k), o['b'],
                                         o['stride'], o['pad'], groups=C), o['relu'])
        return 'dwconv s%d' % o['stride'], kr.worst_ratio(taps[o['out']][:batch, ..., :C], ref,
                                                          kr.bf16_bound(ref, mag, k * k))
    assert kind == 'conv'
    ref, mag = kr.conv_ref(a_in(o['in'], 0, o['c_in']), kr.bf16_round(o['w']), o['b'], o['stride'], o['pad'])
    res = None if o['residual'] < 0 else a_in(o['residual'], 0, o['n_out'])
    ref, mag = epilogue(ref, mag, o['relu'], res)
    return ('conv residual' if res is not None else 'conv'), kr.worst_ratio(
        taps[o['out']][:batch, ..., :o['n_out']], ref, kr.bf16_bound(ref, mag, o['c_in']))


@pytest.mark.parametrize('H,W,B', [(641, 641, 2), (353, 481, 3)])
def test_network_teacher_forced_and_against_fp32(H, W, B):
    shell = mm.make_pose_shell(seed=4)
    plan = network.plan_from_shell(shell)
    tensors, ops, _ = network.build_ops(plan, H, W)
    net = network.CompiledNet(plan, H, W, B)
    images = np.random.default_rng(9).standard_normal((B, 3, H, W)).astype(np.float32)
    x = torch.from_numpy(images).cuda()
    got = [t.clone() for t in net.forward(x)]
    torch.cuda.synchronize()
    taps = {t: net.tap(t, B) for t in range(len(tensors))}
    heads = [t.cpu().numpy() for t in got]
    worst = {}
    for i, o in enumerate(ops):
        kind, r = op_check(o, taps, heads, images, B)
        worst[kind] = max(worst.get(kind, 0.0), r)
        record(kind + ' (mobilenetv2)', r, f'op {i}')
    print(H, W, {k: round(v, 3) for k, v in worst.items()})
    # no 1x1 -> depthwise pair is fused: every depthwise op is its own launch (kind 2), nothing runs as kind 3
    _, kind, _, _ = net.forward_timed(x)
    assert sorted(set(kind.tolist())) == [0, 1, 2] and int((kind == 2).sum()) == 17
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


def test_gemm_impl_1_matches_emulation():
    """the SIMT debug schedule of the whole net equals the bf16 emulation as the wgmma / TMA one does"""
    shell = mm.make_pose_shell(seed=6)
    plan = network.plan_from_shell(shell)
    size, batch = 97, 2
    x = torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(6))
    tensors, ops, _ = network.build_ops(plan, size, size)
    emu_heads, _ = mm.run_ops(tensors, ops, x, bf16=True)
    net = network.CompiledNet(plan, size, size, batch)
    fields = {}
    for impl in (0, 1):
        fields[impl] = [h.cpu().clone() for h in net.forward(x.cuda(), gemm_impl=impl)]
        for hg, he in zip(fields[impl], emu_heads):
            assert float((hg - he).abs().max()) < 5e-2 * max(float(he.abs().max()), 1.0)
    net.close()


def test_predictor_from_shell_equals_cifcaf_on_the_compiled_fields():
    shell = mm.calibrate_pose_heads(mm.make_pose_shell(seed=5))
    pred = predictor.from_shell(shell, 161, 161, 4)
    assert pred.net.heads[0]['stride'] == 32 and (pred.net.heads[0]['h'], pred.net.heads[0]['w']) == (6, 6)
    images = torch.randn(4, 3, 161, 161, generator=torch.Generator().manual_seed(3)).pin_memory()
    sk = torch.tensor(shell.head_nets[1].meta.skeleton, dtype=torch.int64) - 1
    total = 0
    for b in (4, 3):
        res = pred.batch(images[:b])
        cif, caf = pred.fields_batch(images[:b].cuda())
        want = decoder.CifCaf(17, sk).decode_batch(cif, 32, caf, 32)
        assert len(res) == len(want) == b
        for (a, i), (wa, wi) in zip(res, want):
            assert torch.equal(a, wa) and torch.equal(i, wi)
            total += int(a.shape[0])
    print('annotations', total)
    pred.close()


def test_det_predictor_from_shell_equals_cifdet_on_the_compiled_fields():
    shell = det_models.calibrate_det_head(det_models.make_det_shell(mm.MobileNetV2(), 91, 1, seed=2))
    pred = predictor.from_shell(shell, 161, 161, 3)
    assert isinstance(pred, predictor.DetPredictor)
    images = torch.randn(3, 3, 161, 161, generator=torch.Generator().manual_seed(4)).pin_memory()
    res = pred.batch(images)
    (field,) = pred.fields_batch(images.cuda())
    assert tuple(field.shape) == (3, 91, 6, 6, 6)
    want = decoder.CifDet(91).decode_batch(field, 32, nms=True)
    assert len(res) == len(want) == 3
    for (c, s, bx), (wc, ws, wb) in zip(res, want):
        assert torch.equal(c, wc) and torch.equal(s, ws) and torch.equal(bx, wb)
    pred.close()


# ---------------------------------------------------------------------------------------------------- plugin
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
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED
    basenetworks.MobileNetV2.pretrained = False       # no checkpoint can be downloaded
    factory.BASE_FACTORIES['mobilenetv2'] = lambda: basenetworks.MobileNetV2(
        'mobilenetv2', lambda pretrained: torchvision.models.mobilenet_v2(weights=None))
    sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
    import mobilenetv2_models

    torch.manual_seed(0)
    openpifpaf.network.Factory.base_name = 'mobilenetv2'
    openpifpaf.network.Factory.checkpoint = None
    datamodule = openpifpaf.plugins.coco.CocoKp()
    predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas)
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
    print('PLUGIN_MOBILENETV2_OK', json.dumps({'annotations': total}))
''')


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
def test_reference_predictor_runs_mobilenetv2_through_the_plugin(tmp_path):
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', SCRIPT, ROOT], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=900)
    assert 'PLUGIN_MOBILENETV2_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
