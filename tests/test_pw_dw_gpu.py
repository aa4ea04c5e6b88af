"""GPU: the fused 1x1 -> stride-2 depthwise kernel (k_pw_dw) against the two-kernel schedule it replaces
(PIFPAF_FUSE_PW_DW=0) and against the float64 references of tests/kernel_refs.py.

k_pw_dw recomputes the stage-entry 1x1 conv on each depthwise input window with the k16 steps and epilogue of
k_gemm_wg and runs the depthwise FMA loop of k_dwconv5_tma on the result, so every output -- and the elided 1x1 output,
which pifpaf_net_tap_tensor recomputes on demand -- must equal the two-kernel schedule bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

import kernel_refs as kr
from openpifpaf_b200 import _lib, network

pytestmark = pytest.mark.gpu


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def elided_ops(net, x):
    ms, kind, flops, nbytes = net.forward_timed(x)
    return [i for i in range(len(ms)) if kind[i] == 3 and flops[i] == 0 and nbytes[i] == 0 and ms[i] < 0.05], flops


@pytest.mark.parametrize('base,layout,H,W,B,max_batch', [
    ('shufflenetv2k16', 'bins', 337, 401, 3, 4),
    ('shufflenetv2k16', 'shuffle', 97, 129, 2, 2),
    ('shufflenetv2k30', 'bins', 97, 129, 3, 5),
    ('shufflenetv2k30', 'shuffle', 337, 401, 2, 2),
])
def test_fused_net_equals_two_kernels_bitwise(monkeypatch, base, layout, H, W, B, max_batch):
    """head fields and every tensor (the elided 1x1 output too) of the fused and the two-kernel schedules, at sizes
    with partial edge tiles in both directions, batch < max_batch and more items per CTA than the window ring holds"""
    plan = network.random_plan(base, seed=3)
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(4)).cuda()
    nets, heads, elided, flops = {}, {}, {}, {}
    for fuse in ('1', '0'):
        monkeypatch.setenv('PIFPAF_FUSE_PW_DW', fuse)
        net = network.CompiledNet(plan, H, W, max_batch, layout=layout)
        elided[fuse], flops[fuse] = elided_ops(net, x)
        heads[fuse] = [t.clone() for t in net.forward(x)]
        torch.cuda.synchronize()
        nets[fuse] = net
    assert len(elided['1']) == 1 and elided['0'] == []
    assert float(flops['1'].sum()) == float(flops['0'].sum())
    for a, b in zip(heads['1'], heads['0']):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b), float((a - b).abs().max())
    for t in range(len(nets['1'].tensor_shapes)):
        np.testing.assert_array_equal(nets['1'].tap(t, B), nets['0'].tap(t, B), err_msg=f'tensor {t}')
    for net in nets.values():
        net.close()


class PairNet:
    """A net of the two ops alone: tensor 0 (the 1x1 input, K channels) -> conv1x1 (ReLU) -> tensor 1 (pitch mid_c)
    -> depthwise 5x5, stride 2, pad 2 -> tensor 2."""

    def __init__(self, H, W, K, N, mid_c, max_batch, seed, bias_shift):
        rng = np.random.default_rng(seed)
        self.H, self.W, self.K, self.N, self.mid_c, self.mb = H, W, K, N, mid_c, max_batch
        self.C = (N + 15) // 16 * 16
        self.Ho, self.Wo = kr.out_hw(H, W, 5, 2, 2)
        self.x = kr.random_bf16(rng, (max_batch, H, W, K))
        self.w1 = kr.random_bf16(rng, (N, K), 1.0 / np.sqrt(K))
        # large positive 1x1 biases: relu(bias) is far from 0, so a window pixel outside the image that is not
        # written as 0 changes the border outputs
        self.b1 = (rng.standard_normal(N) + bias_shift).astype(np.float32)
        self.dw = (rng.standard_normal((self.C, 25)) * 0.2).astype(np.float32)
        self.dw[N:] = 0.0
        self.db = rng.standard_normal(self.C).astype(np.float32)
        self.db[N:] = 0.0

    def run(self, batch, sm_limit=0):
        L = _lib.lib()
        net = ctypes.c_void_p()
        _lib.check(L.pifpaf_net_create(ctypes.byref(net), 0, self.mb))
        try:
            shapes = [(self.H, self.W, self.K), (self.H, self.W, self.mid_c), (self.Ho, self.Wo, self.C)]
            tid = ctypes.c_int32()
            for h, w, c in shapes:
                _lib.check(L.pifpaf_net_tensor(net, h, w, c, ctypes.byref(tid)))
            _lib.check(L.pifpaf_net_set_tensor(net, 0, self.mb, ptr(self.x), self.x.size))
            _lib.check(L.pifpaf_net_conv1x1(net, 0, 0, self.K, self.N, ptr(self.w1), ptr(self.b1), 1, 1, 0, -1, 0))
            _lib.check(L.pifpaf_net_dwconv(net, 1, 0, self.C, 5, 2, 2, ptr(self.dw), ptr(self.db), 0, 2, 0))
            if sm_limit:
                _lib.check(L.pifpaf_net_set_sm_limit(net, sm_limit))
            _lib.check(L.pifpaf_net_forward(net, None, batch, 0, None))
            torch.cuda.synchronize()
            taps = []
            for h, w, c in shapes[1:]:
                out = np.empty((batch, h, w, c), dtype=np.float32)
                _lib.check(L.pifpaf_net_tap_tensor(net, len(taps) + 1, batch, ptr(out), out.size))
                taps.append(out)
        finally:
            L.pifpaf_net_destroy(net)
        return taps


@pytest.mark.parametrize('H,W,batch,max_batch', [(17, 17, 1, 2), (97, 129, 3, 4), (40, 72, 2, 2)])
def test_pair_borders_schedules_and_float64_bound(monkeypatch, H, W, batch, max_batch):
    """the 1x1 (K = 32, N = 174, the k16 stage-2 entry) -> depthwise pair alone: fused in every launch schedule
    (SM limits, PDL off) == the two-kernel schedule bit for bit, with 1x1 biases large enough that a wrong padding
    rule shows at the borders (17 x 17: the single output tile touches all four); the 1x1 output meets the float64
    bound of the GEMM, the depthwise output the bound of the depthwise conv of that bf16 intermediate"""
    pair = PairNet(H, W, 32, 174, 192, max_batch, seed=H, bias_shift=4.0)
    monkeypatch.setenv('PIFPAF_FUSE_PW_DW', '0')
    want = pair.run(batch)
    schedules = [('1', '1', 0), ('1', '1', 1), ('1', '1', 7), ('1', '1', n_sm() - 4), ('1', '0', 0)]
    for fuse, pdl, sm in schedules:
        monkeypatch.setenv('PIFPAF_FUSE_PW_DW', fuse)
        monkeypatch.setenv('PIFPAF_PDL', pdl)
        got = pair.run(batch, sm_limit=sm)
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g, w, err_msg=f'fuse={fuse} pdl={pdl} sm_limit={sm}')
    mid, out = want
    ref1, mag1 = kr.conv_ref(pair.x[:batch], pair.w1[:, :, None, None], pair.b1, 1, 0)
    ref1, mag1 = kr.epilogue(ref1, mag1, True)
    assert kr.worst_ratio(mid[..., :pair.N], ref1, kr.bf16_bound(ref1, mag1, pair.K)) <= 1.0
    ref2, mag2 = kr.conv_ref(mid[..., :pair.C], pair.dw.reshape(pair.C, 1, 5, 5), pair.db, 2, 2, groups=pair.C)
    assert kr.worst_ratio(out, ref2, kr.bf16_bound(ref2, mag2, 25)) <= 1.0
