"""GPU: the kernels behind the Resnet variants of tests/test_resnet_variants.py -- dilated implicit-GEMM convs
(--resnet-block5-dilation) against float64 with the bound, sentinels and column windows of tests/test_kernels_gpu.py;
k_maxpool (--resnet-pool0-stride) bit for bit against torch.max_pool2d; whole resnet18 variants and the
resnet18-cocodet recipe against fp32 PyTorch and op by op against the bf16 emulation."""
import numpy as np
import pytest
import torch

import det_models
import kernel_refs as kr
import resnet_ops_emulator
from openpifpaf_b200 import _lib, network
from test_kernels_gpu import Case, Check, n_sm, pad8, pad16, ptr

pytestmark = pytest.mark.gpu

FIELD_TOL_REL = 3e-2        # tests/test_network_gpu.py


def dilate(w, d):
    """a k x k kernel with dilation d as the equivalent (d (k - 1) + 1)^2 kernel with zero taps"""
    n, c, k, _ = w.shape
    out = np.zeros((n, c, d * (k - 1) + 1, d * (k - 1) + 1), dtype=w.dtype)
    out[:, :, ::d, ::d] = w
    return out


# (H, W, c_in, dilation, pad, n_out, in_off, residual col (None: no residual), relu, out_off, batch, max_batch)
DIL_CASES = [
    (7, 7, 64, 2, 2, 64, 0, None, 1, 0, 1, 2),           # smaller than one 8 x 16 patch
    (7, 7, 64, 4, 4, 64, 0, 0, 1, 0, 2, 3),              # every tap but the centre row / column in the padding
    (9, 13, 128, 4, 4, 96, 8, 16, 1, 0, 2, 3),
    (17, 19, 72, 2, 2, 80, 0, None, 0, 16, 2, 3),        # K tail, column windows, partial tiles
    (13, 15, 64, 2, 0, 32, 0, None, 1, 0, 1, 2),         # pad 0: the output shrinks by d (k - 1)
    (21, 41, 256, 2, 2, 256, 0, 0, 1, 0, 2, 3),
    (41, 41, 512, 2, 2, 512, 0, 0, 1, 0, 1, 2),          # block5 of resnet18-cocodet at 641 px
    (41, 41, 512, 4, 4, 512, 0, None, 1, 0, 1, 2),
    (81, 81, 64, 2, 2, 64, 0, 0, 1, 0, 1, 2),
    (81, 81, 128, 4, 4, 120, 0, None, 0, 0, 2, 2),
]


def dil_id(c):
    return 'H%dW%d-cin%d-d%dp%d-N%d-in%d-res%s-relu%d-out%d-B%dof%d' % c


def dil_case(H, W, c_in, d, pad, N, in_off, res_col, relu, out_off, batch, mb, seed=0):
    k = 3
    Ho, Wo = kr.out_hw(H, W, d * (k - 1) + 1, 1, pad)
    tensors = [(H, W, pad16(in_off + c_in + 8)), (Ho, Wo, pad16(out_off + pad8(N) + 16))]
    inputs = {0}
    if res_col is not None:
        tensors.append((Ho, Wo, pad16(res_col + N + 8)))
        inputs.add(2)
    case = Case(mb, tensors, inputs=inputs, seed=seed)
    rng = np.random.default_rng(seed + 3)
    w = kr.random_bf16(rng, (N, c_in, k, k), 1 / np.sqrt(c_in * k * k))
    b = rng.standard_normal(N).astype(np.float32)

    def emit(L, net):
        _lib.check(L.pifpaf_net_conv_dilated(net, 0, in_off, c_in, k, 1, pad, N, ptr(w), ptr(b), relu, 1, out_off,
                                             -1 if res_col is None else 2, 0 if res_col is None else res_col, d))

    ref, mag = kr.conv_ref(case.data[0][:batch, ..., in_off:in_off + c_in], dilate(w, d), b, 1, pad)
    res = None if res_col is None else case.data[2][:batch, ..., res_col:res_col + N]
    ref, mag = kr.epilogue(ref, mag, relu, res)
    chk = Check('conv k3 dilated', batch)
    chk.own(1, out_off, out_off + pad8(N))
    chk.compare(1, out_off, ref, kr.bf16_bound(ref, mag, c_in * k * k))
    if res_col is None and pad8(N) > N:
        chk.exact(1, out_off + N, np.zeros(ref.shape[:-1] + (pad8(N) - N,)))
    return case, emit, chk


# the wgmma path at every case, the SIMT debug path at the ones it runs in a few seconds
DIL_PARAMS = [(c, 0) for c in DIL_CASES] + [(c, 1) for c in DIL_CASES if c[0] * c[1] * c[2] * c[5] <= 21 * 41 * 256 * 256]


@pytest.mark.parametrize('c,impl', DIL_PARAMS, ids=lambda v: dil_id(v) if isinstance(v, tuple) else ['wgmma', 'simt'][v])
def test_dilated_conv_matches_float64(c, impl):
    case, emit, chk = dil_case(*c)
    taps, _ = case.run(emit, c[10], impl=impl)
    print(dil_id(c), impl, '%.3f' % chk.verify(taps, dil_id(c)))


@pytest.mark.parametrize('c', [DIL_CASES[2], DIL_CASES[5], DIL_CASES[8]], ids=dil_id)
def test_dilated_conv_schedules_are_bitwise_invariant(c, monkeypatch):
    """the persistent grid at SM limits 1 / 7 / n_sm - 4 and without programmatic dependent launch"""
    case, emit, _ = dil_case(*c)
    want, _ = case.run(emit, c[10])
    for lim in (1, 7, n_sm() - 4):
        got, _ = case.run(emit, c[10], sm_limit=lim)
        assert np.array_equal(got[1], want[1]), lim
    monkeypatch.setenv('PIFPAF_PDL', '0')
    got, _ = case.run(emit, c[10])
    assert np.array_equal(got[1], want[1])


def test_dilated_conv_rejects_stride_2():
    L = _lib.lib()
    case = Case(1, [(9, 9, 64), (5, 5, 64)], inputs={0})
    w = np.zeros((64, 64, 3, 3), dtype=np.float32)
    b = np.zeros(64, dtype=np.float32)

    def emit(L, net):
        rc = L.pifpaf_net_conv_dilated(net, 0, 0, 64, 3, 2, 2, 64, ptr(w), ptr(b), 1, 1, 0, -1, 0, 2)
        assert rc != 0
        assert 'stride 1' in L.pifpaf_last_error().decode()
    case.run(emit, 1)


# (H, W, channels, stride, in_off, out_off, batch, max_batch)
POOL_CASES = [
    (1, 1, 16, 2, 0, 0, 1, 2),
    (2, 3, 16, 1, 0, 0, 2, 3),
    (7, 9, 24, 2, 8, 0, 2, 3),
    (8, 10, 64, 2, 0, 16, 1, 2),
    (9, 11, 20, 2, 0, 0, 2, 3),           # 20 channels: the padding columns of the 8-channel vector pass through
    (8, 10, 64, 1, 0, 0, 3, 4),
    (33, 31, 64, 2, 0, 0, 2, 3),
    (161, 161, 64, 2, 0, 0, 2, 2),        # the stem output of a 321 px image
    (40, 41, 200, 1, 16, 8, 2, 3),
    (17, 16, 512, 2, 0, 0, 2, 3),
    (17, 16, 512, 1, 0, 0, 1, 2),
]


def pool_id(c):
    return 'H%dW%d-C%d-s%d-in%d-out%d-B%dof%d' % c


@pytest.mark.parametrize('c', POOL_CASES, ids=pool_id)
def test_maxpool_equals_torch_bitwise(c):
    H, W, C, s, in_off, out_off, batch, mb = c
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    case = Case(mb, [(H, W, pad16(in_off + C + 8)), (Ho, Wo, pad16(out_off + pad8(C) + 8))], inputs={0})

    def emit(L, net):
        _lib.check(L.pifpaf_net_maxpool(net, 0, in_off, C, s, 1, out_off))

    x = torch.from_numpy(case.data[0][:batch, ..., in_off:in_off + C]).cuda().to(torch.bfloat16).permute(0, 3, 1, 2)
    want = torch.max_pool2d(x, 3, s, 1).permute(0, 2, 3, 1).float().cpu().numpy()
    taps, _ = case.run(emit, batch)
    chk = Check('maxpool', batch)
    chk.own(1, out_off, out_off + pad8(C))
    chk.exact(1, out_off, want)
    if pad8(C) > C:         # padding columns of the input window hold random values: the pool passes them through
        chk.exact(1, out_off + C, torch.max_pool2d(
            torch.from_numpy(case.data[0][:batch, ..., in_off + C:in_off + pad8(C)]).permute(0, 3, 1, 2), 3, s, 1
        ).permute(0, 2, 3, 1).numpy())
    assert chk.verify(taps, pool_id(c)) == 0.0


def test_maxpool_reports_its_own_op_kind():
    plan = network.random_resnet_plan('resnet18', pool0_stride=2, seed=0)
    net = network.CompiledNet(plan, 97, 97, 1)
    x = torch.randn(1, 3, 97, 97).cuda()
    _, kind, flops, _ = net.forward_timed(x)
    assert list(kind[:2]) == [0, 4] and flops[1] == 0
    assert (kind[2:-1] == 1).all()


@pytest.mark.parametrize('variant', list(det_models.VARIANTS))
def test_resnet18_variant_matches_emulation_and_fp32(variant):
    shell = det_models.make_variant_shell(variant, seed=4)
    plan = network.plan_from_shell(shell)
    size, batch = 161, 2
    x = torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(6))
    tensors, ops, _ = network.build_ops(plan, size, size)
    emu_heads, emu_acts = resnet_ops_emulator.run_ops(tensors, ops, x, bf16=True)
    net = network.CompiledNet(plan, size, size, batch)
    for impl in (1, 0):
        heads = net.forward(x.cuda(), gemm_impl=impl)
        torch.cuda.synchronize()
        for o in ops:
            if o['kind'] == 'heads':
                continue
            got = net.tap(o['out'], batch)
            ref = emu_acts[o['out']].numpy()
            scale = max(float(np.abs(ref).max()), 1e-6)
            assert float(np.abs(got - ref).max()) / scale < 3e-2, (impl, o['kind'], o['out'], o.get('dilation'))
        for hg, he in zip(heads, emu_heads):
            assert hg.shape == he.shape
            assert float((hg.cpu() - he).abs().max()) < 5e-2 * max(float(he.abs().max()), 1.0)
    with torch.no_grad():
        want = shell(x)
    for hg, hw_ in zip(net.forward(x.cuda()), want):
        assert hg.shape == hw_.shape
        err = (hg.cpu() - hw_).abs()
        assert float(err.max()) < FIELD_TOL_REL * float(hw_.std()) + 1e-3
        assert float(err.mean()) < 1e-2 * float(hw_.std())


def test_cocodet_recipe_at_641_matches_fp32():
    """the resnet18-cocodet recipe at the size the benchmark of detection models uses: 91 x 6 x 81 x 81 fields"""
    shell = det_models.make_variant_shell('cocodet', seed=5)
    net = network.CompiledNet(network.plan_from_shell(shell), 641, 641, 2)
    x = torch.randn(2, 3, 641, 641, generator=torch.Generator().manual_seed(2)).cuda()
    (got,) = net.forward(x)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        (want,) = shell.cuda()(x)
    assert got.shape == want.shape == (2, 91, 6, 81, 81)
    err = (got - want).abs()
    assert float(err.max()) < FIELD_TOL_REL * float(want.std()) + 1e-3
