"""GPU: a net compiled at a capacity and run at a smaller size (`CompiledNet.set_input_size`) computes, bit for bit, what
a net compiled at exactly that size computes -- every head field and every tapped tensor -- for every plan family,
through the float and the uint8 stem, on the tensor-core and the SIMT GEMM routes, without the fused 1x1 -> depthwise
kernel, across alternating sizes and batches on one net, and after refused sizes."""
import ctypes

import numpy as np
import pytest
import torch

import input_size_models as ism
from openpifpaf_b200 import _lib, network

pytestmark = pytest.mark.gpu

CAP = (161, 193)
MAX_BATCH = 3


def _features(net, b, seed):
    h, w, _ = net.tensor_shapes[0]
    c = net.op_desc[0]['k_cols']
    g = torch.Generator().manual_seed(seed)
    return torch.randn((b, h, w, c), generator=g).numpy()


def run(net, b, seed, gemm_impl=0, uint8=False):
    """fields and every tensor of one forward of b seeded images at the net's current size"""
    h, w = net.input_size
    g = torch.Generator().manual_seed(seed)
    if net.op_desc[0]['kind'] == 'heads':
        heads = net.forward_features(_features(net, b, seed), gemm_impl=gemm_impl)
    elif uint8:
        x = torch.randint(0, 256, (b, h, w, 3), generator=g, dtype=torch.uint8).cuda()
        heads = net.forward_uint8(x, gemm_impl=gemm_impl)
    else:
        heads = net.forward(torch.randn((b, 3, h, w), generator=g).cuda(), gemm_impl=gemm_impl)
    torch.cuda.synchronize()
    fields = [t.cpu().numpy().copy() for t in heads]
    return fields, [net.tap(t, b) for t in range(len(net.tensor_shapes))]


def assert_same(got, want, what):
    (gf, gt), (wf, wt) = got, want
    assert len(gf) == len(wf)
    for i, (a, b) in enumerate(zip(gf, wf)):
        assert a.shape == b.shape, (what, 'head', i, a.shape, b.shape)
        np.testing.assert_array_equal(a, b, err_msg=f'{what}: head {i}')
    for t, (a, b) in enumerate(zip(gt, wt)):
        assert a.shape == b.shape, (what, 'tensor', t, a.shape, b.shape)
        np.testing.assert_array_equal(a, b, err_msg=f'{what}: tensor {t}')


def compiled_at(name, h, w, **kw):
    return network.CompiledNet(ism.plan(name), h, w, MAX_BATCH, **kw)


@pytest.mark.parametrize('name', sorted(ism.FAMILIES))
def test_each_size_equals_a_net_compiled_at_it(name):
    net = compiled_at(name, *CAP)
    heads_only = ism.plan(name)['kind'] == 'heads_only'
    sizes = ism.sizes(*CAP) + [ism.tiny(name)]
    for i, (h, w) in enumerate(sizes):
        ref = compiled_at(name, h, w)
        net.set_input_size(h, w)
        assert net.input_size == (h, w) and net.tensor_shapes == ref.tensor_shapes
        assert [(hd['h'], hd['w']) for hd in net.heads] == [(hd['h'], hd['w']) for hd in ref.heads]
        assert net.flops_per_image == ref.flops_per_image
        if (h, w) == ism.tiny(name):
            assert all((hd['h'], hd['w']) == (1, 1) for hd in net.heads)
        b = 1 + i % MAX_BATCH
        assert_same(run(net, b, i), run(ref, b, i), f'{name} {h}x{w} batch {b}')
        if i % 4 == 0:
            assert_same(run(net, b, i, gemm_impl=1), run(ref, b, i, gemm_impl=1), f'{name} {h}x{w} simt')
        if i % 4 == 1 and not heads_only:
            assert_same(run(net, b, i, uint8=True), run(ref, b, i, uint8=True), f'{name} {h}x{w} uint8')
        ref.close()
    net.close()


def test_without_the_fused_pw_dw_kernel(monkeypatch):
    monkeypatch.setenv('PIFPAF_FUSE_PW_DW', '0')
    net = compiled_at('k16', *CAP)
    for i, (h, w) in enumerate(ism.sizes(*CAP, seed=3)[:6]):
        ref = compiled_at('k16', h, w)
        net.set_input_size(h, w)
        assert_same(run(net, 2, i), run(ref, 2, i), f'PIFPAF_FUSE_PW_DW=0 {h}x{w}')
        ref.close()
    net.close()


@pytest.mark.parametrize('name', ['k16', 'cifdet_up2', 'mobilenetv2'])
def test_alternating_sizes_and_batches(name):
    """A, B, A, B on one net with the batch changing at every step; the store maps follow both"""
    a, b = (97, 130), (161, 65)
    net = compiled_at(name, *CAP)
    refs = {a: compiled_at(name, *a), b: compiled_at(name, *b)}
    for step, (size, batch) in enumerate([(a, 3), (b, 1), (a, 2), (b, 3), (CAP, 1), (a, 1)]):
        ref = refs.setdefault(size, compiled_at(name, *size))
        net.set_input_size(*size)
        assert_same(run(net, batch, step), run(ref, batch, step), f'{name} step {step} {size} batch {batch}')
    net.close()


def _c_set_size(net, h, w, table):
    t = np.ascontiguousarray(np.asarray(table, dtype=np.int32).reshape(-1))
    return net.lib.pifpaf_net_set_input_size(net.handle, h, w, len(t) // 2, t.ctypes.data_as(ctypes.c_void_p))


def test_refused_sizes_leave_the_previous_size():
    net = compiled_at('k16', *CAP)
    size = (100, 120)
    ref = compiled_at('k16', *size)
    net.set_input_size(*size)
    want = run(ref, 2, 0)
    for bad in [(CAP[0] + 1, CAP[1]), (CAP[0], CAP[1] + 16), (0, 50)]:
        with pytest.raises(RuntimeError):
            net.set_input_size(*bad)
        assert net.input_size == size
    # the library's own check: a table a tensor of which exceeds its capacity, or disagrees with an op
    good = [s[:2] for s in network.tensor_shapes_at(net.op_desc, net.capacity_shapes, 64, 64)]
    over = list(good)
    over[-1] = (net.capacity_shapes[-1][0] + 1, over[-1][1])
    wrong = list(good)
    wrong[3] = (wrong[3][0] - 1, wrong[3][1])
    for table in (over, wrong, good[:-1]):
        assert _c_set_size(net, 64, 64, table) == _lib.E_BADARG
    assert _c_set_size(net, CAP[0] + 16, CAP[1], good) == _lib.E_BADARG
    assert [(hd['h'], hd['w']) for hd in net.heads] == [(hd['h'], hd['w']) for hd in ref.heads]
    assert_same(run(net, 2, 0), want, 'after refusals')
    net.close()


def test_a_size_that_empties_a_layer_is_refused():
    plan = network.random_resnet_plan('resnet18', seed=0)
    plan['input']['pad'] = 0             # a 7x7 stem without padding: nothing below 7 pixels
    net = network.CompiledNet(plan, 64, 64, 2)
    ref = network.CompiledNet(plan, 7, 9, 2)
    with pytest.raises(RuntimeError, match='empty output'):
        net.set_input_size(6, 9)
    table = [s[:2] for s in network.tensor_shapes_at(net.op_desc, net.capacity_shapes, 7, 9)]
    assert _c_set_size(net, 6, 9, table) == _lib.E_BADARG
    assert net.input_size == (64, 64)
    net.set_input_size(7, 9)
    assert_same(run(net, 2, 1), run(ref, 2, 1), 'after an empty-layer refusal')
    net.close()


def test_k16_at_641_runs_tight_canvases():
    """the canvases CenterPadTight(16) gives 641-pixel photos of common aspect ratios, on a 641 x 641 net"""
    net = network.CompiledNet(ism.plan('k16'), 641, 641, 2)
    for i, size in enumerate([(481, 641), (641, 481), (433, 641), (641, 369)]):
        ref = network.CompiledNet(ism.plan('k16'), *size, 2)
        net.set_input_size(*size)
        assert_same(run(net, 2, i), run(ref, 2, i), f'641 capacity at {size}')
        ref.close()
    net.close()
