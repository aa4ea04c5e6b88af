"""GPU: the kernel launches of one forward of the shipped networks, against what the op list predicts.

net.cu picks each op's kernels when the op is emitted and the forward only reads that choice. Pinned here, in every
setting that changes a route (gemm_impl 0 and 1, the 'bins' and 'shuffle' layouts, PIFPAF_FUSE_PW_DW=0,
PIFPAF_DW_CBF=1):
- a forward launches one kernel per op, less one per 1x1 -> depthwise pair that k_pw_dw runs (gemm_impl 0 only);
- forward_timed reports each op's kind as the op list and tests/net_plan.py's fused_pairs predict;
- the tensor conversions of tap / set_tensor are one counted launch each;
- the fused depthwise -> 1x1 op (fuse_dw=True) has no SIMT route and is refused at gemm_impl 1."""
import ctypes

import numpy as np
import pytest
import torch

import mobilenetv2_models as mm
import net_plan
from openpifpaf_b200 import _lib, network

pytestmark = pytest.mark.gpu

SIZE, BATCH = 129, 2

# forward_timed's op kinds: 0 input conv, 1 GEMM, 2 depthwise, 3 fused kernels, 4 max pool
KIND = {'input_conv': 0, 'conv1x1': 1, 'conv': 1, 'heads': 1, 'dwconv': 2, 'dw_conv1x1': 3, 'maxpool': 4}

PLANS = {
    'k16': lambda: network.random_plan('shufflenetv2k16', seed=0),
    'k30': lambda: network.random_plan('shufflenetv2k30', seed=0),
    'k16-stride8': lambda: network.random_plan('shufflenetv2k16', seed=0, stage4_dilation=2),
    'r18': lambda: network.random_resnet_plan('resnet18', seed=0),
    'r18-pool0': lambda: network.random_resnet_plan('resnet18', pool0_stride=2, seed=0),
    'r50': lambda: network.random_resnet_plan('resnet50', seed=0),
    'mobilenetv2': lambda: network.plan_from_shell(mm.make_pose_shell(seed=0)),
}
SHUFFLENETS = ('k16', 'k30', 'k16-stride8')
# (layout, environment) of the ShuffleNetV2K nets; the other nets have one lowering and ignore these switches
SETTINGS = {
    'bins': ('bins', {}),
    'shuffle': ('shuffle', {}),
    'no-pw-dw': ('bins', {'PIFPAF_FUSE_PW_DW': '0'}),
    'cbf': ('bins', {'PIFPAF_DW_CBF': '1'}),
    'shuffle-cbf': ('shuffle', {'PIFPAF_DW_CBF': '1'}),
}
CASES = [(n, s) for n in SHUFFLENETS for s in SETTINGS] + [(n, None) for n in PLANS if n not in SHUFFLENETS]


def launches(fn):
    """library kernel launches made by fn()"""
    L = _lib.lib()
    n0 = L.pifpaf_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(L.pifpaf_launch_count() - n0)


def build(monkeypatch, name, setting):
    """the compiled net and its op list; the switches are read when the native net is created"""
    layout, env = SETTINGS[setting] if setting else (None, {})
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    plan = PLANS[name]()
    tensors, ops, _ = network.build_ops(plan, SIZE, SIZE, layout=layout, fuse_dw=False)
    net = network.CompiledNet(plan, SIZE, SIZE, BATCH + 1, layout=layout, fuse_dw=False)
    pairs = net_plan.fused_pairs(tensors, ops, fuse_pw_dw=env.get('PIFPAF_FUSE_PW_DW', '1') != '0')
    return net, ops, pairs


def expected_kinds(ops, pairs):
    kinds = [KIND[o['kind']] for o in ops]
    for i in pairs:
        kinds[i] = kinds[i + 1] = 3
    return kinds


@pytest.mark.parametrize('gemm_impl', [0, 1], ids=['wgmma', 'simt'])
@pytest.mark.parametrize('name,setting', CASES, ids=lambda v: v if v else 'default')
def test_forward_launches_and_timed_kinds(monkeypatch, name, setting, gemm_impl):
    """one launch per op, less the 1x1s k_pw_dw computes (gemm_impl 0); forward_timed's kinds as predicted"""
    net, ops, pairs = build(monkeypatch, name, setting)
    try:
        assert net.num_ops == len(ops)
        if name in SHUFFLENETS:             # the stage-2 entry pair, in either depthwise item order
            assert len(pairs) == (0 if setting == 'no-pw-dw' else 1)
        x = torch.randn(BATCH, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(1)).cuda()
        want = len(ops) - (len(pairs) if gemm_impl == 0 else 0)
        assert launches(lambda: net.forward(x, gemm_impl=gemm_impl)) == want
        timed = []
        assert launches(lambda: timed.append(net.forward_timed(x, gemm_impl=gemm_impl))) == want
        ms, kind, flops, _ = timed[0]
        assert kind.tolist() == expected_kinds(ops, pairs if gemm_impl == 0 else [])
        assert (ms >= 0).all() and float(flops.sum()) == pytest.approx(net.flops_per_image * BATCH)
    finally:
        net.close()


def test_tensor_conversions_are_counted_launches(monkeypatch):
    """tap: one conversion, plus the GEMM of a 1x1 output the last forward kept inside k_pw_dw; set_tensor: one"""
    net, ops, pairs = build(monkeypatch, 'k16', 'bins')
    try:
        x = torch.randn(BATCH, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(2)).cuda()
        net.forward(x)
        torch.cuda.synchronize()
        mid, other = ops[pairs[0]]['out'], ops[0]['out']
        assert launches(lambda: net.tap(mid, BATCH)) == 2
        assert launches(lambda: net.tap(other, BATCH)) == 1
        before = net.tap(other, BATCH)
        data = np.ascontiguousarray(before)
        L = _lib.lib()
        assert launches(lambda: _lib.check(L.pifpaf_net_set_tensor(
            net.handle, other, BATCH, data.ctypes.data_as(ctypes.c_void_p), data.size))) == 1
        np.testing.assert_array_equal(net.tap(other, BATCH), before)
    finally:
        net.close()


def test_fused_depthwise_gemm_is_refused_at_gemm_impl_1():
    """fuse_dw=True: the k_dw_gemm op runs at gemm_impl 0 and is refused at gemm_impl 1"""
    plan = PLANS['k16']()
    tensors, ops, _ = network.build_ops(plan, SIZE, SIZE, fuse_dw=True)
    assert any(o['kind'] == 'dw_conv1x1' for o in ops)
    net = network.CompiledNet(plan, SIZE, SIZE, BATCH, fuse_dw=True)
    try:
        x = torch.randn(BATCH, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(3)).cuda()
        assert launches(lambda: net.forward(x)) == len(ops) - len(net_plan.fused_pairs(tensors, ops))
        with pytest.raises(RuntimeError, match='no SIMT debug variant'):
            net.forward(x, gemm_impl=1)
    finally:
        net.close()
