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
import net_plan
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
    tensors, ops, _ = network.build_ops(plan, H, W, layout=layout)
    assert elided['1'] == net_plan.fused_pairs(tensors, ops) and len(elided['1']) == 1 and elided['0'] == []
    assert float(flops['1'].sum()) == float(flops['0'].sum())
    for a, b in zip(heads['1'], heads['0']):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b), float((a - b).abs().max())
    for t in range(len(nets['1'].tensor_shapes)):
        np.testing.assert_array_equal(nets['1'].tap(t, B), nets['0'].tap(t, B), err_msg=f'tensor {t}')
    for net in nets.values():
        net.close()


class PairNet:
    """A net of the two ops alone: tensor 0 (the 1x1 input: `pitch` channels, K of them read from column in_off) ->
    1x1 conv (N outputs, activation relu1) -> tensor 1 (the intermediate) -> depthwise (C channels from column
    dw_in_off; 5x5, stride 2, pad 2 unless `dw` = (kernel, stride, pad, dilation) says otherwise; ReLU if relu2) ->
    tensor 2.  Every input column holds random bf16 values (the padding columns too: their weights are zero).
    Variants that the fusion must refuse: residual (the 1x1 adds tensor 3), out_off (the 1x1 writes the intermediate
    from that column), third ('read': a max pool reads the intermediate into tensor 3, 'write': a second 1x1 writes
    the columns past the first one's)."""

    def __init__(self, H, W, K, N, C, pitch, relu1, relu2, max_batch, seed, bias_shift=4.0, in_off=0, out_off=0,
                 dw_in_off=0, dw=(5, 2, 2, 1), residual=False, third=None):
        rng = np.random.default_rng(seed)
        self.H, self.W, self.K, self.N, self.C, self.mb = H, W, K, N, C, max_batch
        self.pitch, self.relu1, self.relu2, self.in_off, self.out_off, self.dw_in_off = \
            pitch, relu1, relu2, in_off, out_off, dw_in_off
        self.dw_geom, self.residual, self.third = dw, residual, third
        k, st, pad, dil = dw
        self.mid_c = pad16(max(out_off + pad8(N), dw_in_off + pad8(C)) + (16 if third == 'write' else 0))
        self.Ho, self.Wo = kr.out_hw(H, W, (k - 1) * dil + 1, st, pad)
        self.x = kr.random_bf16(rng, (max_batch, H, W, pitch))
        self.w1 = kr.random_bf16(rng, (N, K), 1.0 / np.sqrt(K))
        # large positive 1x1 biases: relu(bias) is far from 0, so a window pixel outside the image that is not
        # written as 0 changes the border outputs
        self.b1 = (rng.standard_normal(N) + bias_shift).astype(np.float32)
        self.dw = (rng.standard_normal((C, k * k)) * 0.2).astype(np.float32)
        self.db = rng.standard_normal(C).astype(np.float32)
        self.res = kr.random_bf16(rng, (max_batch, H, W, pad16(N))) if residual else None
        self.w3 = kr.random_bf16(rng, (16, K), 1.0 / np.sqrt(K))
        self.shapes = [(H, W, pitch), (H, W, self.mid_c), (self.Ho, self.Wo, pad16(C))]
        if residual:
            self.shapes.append((H, W, pad16(N)))
        elif third == 'read':
            self.shapes.append(((H - 1) // 2 + 1, (W - 1) // 2 + 1, self.mid_c))

    def build(self, L, net):
        tid = ctypes.c_int32()
        for h, w, c in self.shapes:
            _lib.check(L.pifpaf_net_tensor(net, h, w, c, ctypes.byref(tid)))
        _lib.check(L.pifpaf_net_set_tensor(net, 0, self.mb, ptr(self.x), self.x.size))
        if self.residual:
            _lib.check(L.pifpaf_net_set_tensor(net, 3, self.mb, ptr(self.res), self.res.size))
            _lib.check(L.pifpaf_net_conv(net, 0, self.in_off, self.K, 1, 1, 0, self.N, ptr(self.w1), ptr(self.b1),
                                         self.relu1, 1, self.out_off, 3, 0))
        else:
            _lib.check(L.pifpaf_net_conv1x1(net, 0, self.in_off, self.K, self.N, ptr(self.w1), ptr(self.b1),
                                            self.relu1, 1, self.out_off, -1, 0))
        k, st, pad, dil = self.dw_geom
        _lib.check(L.pifpaf_net_dwconv_dilated(net, 1, self.dw_in_off, self.C, k, st, pad, ptr(self.dw), ptr(self.db),
                                               self.relu2, 2, 0, dil))
        if self.third == 'read':
            _lib.check(L.pifpaf_net_maxpool(net, 1, 0, self.mid_c, 2, 3, 0))
        elif self.third == 'write':
            _lib.check(L.pifpaf_net_conv1x1(net, 0, self.in_off, self.K, 16, ptr(self.w3), ptr(self.b1), 1, 1,
                                            self.mid_c - 16, -1, 0))

    def run(self, batch, sm_limit=0):
        """-> (taps of tensors 1.. after one forward, indices of the ops the forward elided)"""
        L = _lib.lib()
        net = ctypes.c_void_p()
        _lib.check(L.pifpaf_net_create(ctypes.byref(net), 0, self.mb))
        try:
            self.build(L, net)
            if sm_limit:
                _lib.check(L.pifpaf_net_set_sm_limit(net, sm_limit))
            _lib.check(L.pifpaf_net_forward(net, None, batch, 0, None))
            torch.cuda.synchronize()
            taps = []
            for t, (h, w, c) in enumerate(self.shapes[1:], 1):
                out = np.empty((batch, h, w, c), dtype=np.float32)
                _lib.check(L.pifpaf_net_tap_tensor(net, t, batch, ptr(out), out.size))
                taps.append(out)
            n = L.pifpaf_net_num_ops(net)
            ms, kind = np.zeros(n, dtype=np.float32), np.zeros(n, dtype=np.int32)
            flops, nbytes = np.zeros(n), np.zeros(n)
            _lib.check(L.pifpaf_net_forward_timed(net, None, batch, 0, None, ptr(ms), ptr(kind), ptr(flops),
                                                  ptr(nbytes)))
            elided = [i for i in range(n) if kind[i] == 3 and flops[i] == 0 and nbytes[i] == 0]
        finally:
            L.pifpaf_net_destroy(net)
        return taps, elided

    def plan_ops(self):
        """the two ops as network.build_ops dicts (tests/net_plan.py's input)"""
        k, st, pad, dil = self.dw_geom
        g = {'kind': 'conv1x1', 'in': 0, 'in_off': self.in_off, 'k_cols': self.K, 'n_out': self.N,
             'relu': self.relu1, 'out': 1, 'out_off': self.out_off, 'shuffle_src': -1}
        if self.residual:
            g = {'kind': 'conv', 'in': 0, 'in_off': self.in_off, 'c_in': self.K, 'kernel': 1, 'stride': 1, 'pad': 0,
                 'n_out': self.N, 'relu': self.relu1, 'out': 1, 'out_off': self.out_off, 'residual': 3}
        d = {'kind': 'dwconv', 'in': 1, 'in_off': self.dw_in_off, 'channels': self.C, 'kernel': k, 'stride': st,
             'pad': pad, 'dilation': dil, 'relu': self.relu2, 'out': 2}
        return g, d

    def refusal(self):
        g, d = self.plan_ops()
        return net_plan.pw_dw_refusal(g, d, self.pitch, others_touch_mid=self.third is not None)

    def check_float64(self, batch, mid, out):
        """both stages against their float64 bounds: the 1x1 output, and the depthwise conv of that bf16 intermediate"""
        ref1, mag1 = kr.conv_ref(self.x[:batch, ..., self.in_off:self.in_off + self.K], self.w1[:, :, None, None],
                                 self.b1, 1, 0)
        res = self.res[:batch, ..., :self.N] if self.residual else None
        ref1, mag1 = kr.epilogue(ref1, mag1, self.relu1, res)
        r1 = kr.worst_ratio(mid[..., self.out_off:self.out_off + self.N], ref1, kr.bf16_bound(ref1, mag1, self.K))
        k, st, pad, dil = self.dw_geom
        C = self.C
        ref2, mag2 = kr.conv_ref(mid[..., self.dw_in_off:self.dw_in_off + C], self.dw.reshape(C, 1, k, k), self.db,
                                 st, pad, groups=C, dilation=dil)
        ref2, mag2 = kr.epilogue(ref2, mag2, self.relu2)
        r2 = kr.worst_ratio(out[..., :C], ref2, kr.bf16_bound(ref2, mag2, k * k))
        assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
        # channels past N / C: zero weights and biases (the 8-channel tails) or never written (the 16-channel pitch)
        pad_out = self.out_off + self.N
        assert (mid[..., pad_out:pad16(pad_out)] == 0).all() and (out[..., C:] == 0).all()
        return r1, r2


def pad8(v):
    return (v + 7) // 8 * 8


def pad16(v):
    return (v + 15) // 16 * 16


# (H, W, K, N, C, input pitch, relu1, relu2, batch, max_batch): the domain plan_pw_dw admits -- K <= 32 in an input
# of pitch 16 or 32 (the 32-channel window box wider than a 16-channel tensor), 1 to 5 depthwise channel blocks (320
# channels: 231 296 bytes of shared memory, the last width that fits), a depthwise reading fewer channels than the 1x1
# writes, both activations on and off; 17 x 17 and 15 x 16: one output tile touching all four borders; 161 x 161 and
# more images: many tiles per CTA
PAIR_CASES = [
    (17, 17, 32, 174, 174, 32, 1, 0, 1, 2),       # the k16 stage-2 entry
    (97, 129, 32, 174, 174, 32, 1, 0, 3, 4),
    (40, 72, 32, 174, 174, 32, 1, 0, 2, 3),
    (17, 17, 8, 8, 8, 16, 1, 1, 1, 2),            # 1 channel block, 8 channels
    (15, 16, 16, 64, 64, 16, 0, 0, 2, 3),
    (33, 31, 24, 72, 72, 32, 1, 1, 2, 3),         # 2 blocks
    (18, 21, 8, 176, 176, 32, 0, 1, 1, 2),
    (40, 39, 16, 256, 256, 16, 1, 0, 2, 3),       # 4 blocks, 16-channel input
    (35, 33, 32, 320, 320, 32, 0, 1, 2, 3),       # 5 blocks: the shared-memory edge
    (16, 18, 24, 320, 320, 32, 1, 1, 1, 2),
    (29, 30, 32, 176, 64, 32, 1, 0, 2, 3),        # the depthwise reads 64 of the 176 channels
    (161, 161, 16, 320, 320, 16, 1, 1, 2, 3),
]


def pair_id(c):
    return 'H%dW%d-K%d-N%d-C%d-pitch%d-relu%d%d-B%dof%d' % c


@pytest.mark.parametrize('c', PAIR_CASES, ids=pair_id)
def test_pair_borders_schedules_and_float64_bound(monkeypatch, c):
    """the 1x1 -> depthwise pair alone: fused (one k_pw_dw launch) in every launch schedule (SM limits, PDL off) ==
    the two-kernel schedule bit for bit -- the depthwise output and the elided intermediate, which the tap recomputes
    -- with 1x1 biases large enough that a wrong padding rule shows at the borders; the 1x1 output meets the float64
    bound of the GEMM, the depthwise output the bound of the depthwise conv of that bf16 intermediate"""
    H, W, K, N, C, pitch, relu1, relu2, batch, mb = c
    pair = PairNet(H, W, K, N, C, pitch, relu1, relu2, mb, seed=H + N)
    assert pair.refusal() is None
    monkeypatch.setenv('PIFPAF_FUSE_PW_DW', '0')
    want, elided = pair.run(batch)
    assert elided == []
    schedules = [('1', '1', 0), ('1', '1', 1), ('1', '1', 7), ('1', '1', n_sm() - 4), ('1', '0', 0)]
    for fuse, pdl, sm in schedules:
        monkeypatch.setenv('PIFPAF_FUSE_PW_DW', fuse)
        monkeypatch.setenv('PIFPAF_PDL', pdl)
        got, elided = pair.run(batch, sm_limit=sm)
        assert elided == [0], elided
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g, w, err_msg=f'fuse={fuse} pdl={pdl} sm_limit={sm}')
    print(pair_id(c), 'err / bound %.3f %.3f' % pair.check_float64(batch, *want))


# planner rule -> PairNet keywords of a pair that rule alone refuses
RULE_CASES = {
    'residual': dict(residual=True),
    'ReLU6': dict(relu1=2),
    'input wider than PWDW_K': dict(pitch=48),
    'input column offset': dict(pitch=32, K=16, in_off=16),
    'output column offset': dict(out_off=16),
    'depthwise pad': dict(dw=(5, 2, 1, 1)),
    'depthwise 3x3': dict(dw=(3, 2, 1, 1)),
    'depthwise stride 1': dict(dw=(5, 1, 2, 1)),
    'depthwise dilated': dict(dw=(5, 1, 4, 2)),
    'depthwise input column offset': dict(dw_in_off=16),
    'another op reads the intermediate': dict(third='read'),
    'another op writes the intermediate': dict(third='write'),
    'shared memory': dict(N=328, C=328),
}
RULE_REASON = {'depthwise 3x3': 'depthwise is not the TMA 5x5 stride-2 kernel',
               'depthwise stride 1': 'depthwise is not the TMA 5x5 stride-2 kernel',
               'depthwise dilated': 'depthwise is not the TMA 5x5 stride-2 kernel',
               'another op reads the intermediate': 'another op touches the intermediate',
               'another op writes the intermediate': 'another op touches the intermediate'}


def rule_pair(rule):
    kw = dict(H=19, W=23, K=24, N=72, C=72, pitch=32, relu1=1, relu2=0, max_batch=3, seed=5)
    kw.update(RULE_CASES[rule])
    return PairNet(**kw)


@pytest.mark.parametrize('rule', list(RULE_CASES))
def test_planner_rule_refuses_the_pair(monkeypatch, rule):
    """each rule of plan_pw_dw alone keeps the pair two launches (forward_timed elides nothing), as tests/net_plan.py
    predicts, and the two ops still meet their float64 bounds"""
    pair = rule_pair(rule)
    assert pair.refusal() == RULE_REASON.get(rule, rule)
    monkeypatch.setenv('PIFPAF_FUSE_PW_DW', '1')
    (mid, out, *_), elided = pair.run(2)
    assert elided == []
    print(rule, 'err / bound %.3f %.3f' % pair.check_float64(2, mid, out))
