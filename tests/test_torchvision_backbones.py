"""CPU: the torchvision-backed base networks of the reference -- ShuffleNetV2 x1 / x2 (basenetworks.py:36-68) and
SqueezeNet 1.1 (basenetworks.py:461-499).  (1) The test mirror in torchvision_backbone_models.py equals the reference's
own modules (stored features at an odd and an even size, and the live modules where the reference sources exist); (2)
the product's plan and lowering reproduce the fp32 Shell in the CPU interpreter (both ShuffleNet layouts) and stay
within the field tolerance in the bf16 emulation; (3) the ceil-mode size rule equals torch's; (4) the per-size tensor
table equals the lowering at each size; (5) the kernels net.cu's planner picks for these nets; (6) the variants the
compiled forward does not implement are refused, MobileNetV3 still with its Hardswish message."""
import contextlib
import functools
import os
import types
from unittest import mock

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers
import input_size_models as ism
import kernel_refs as kr
import net_plan
import ops_emulator
import torchvision_backbone_models as tbm
from openpifpaf_b200 import network
from oracle import build_ref

HAVE_REF_SRC = os.path.isdir(build_ref.REF_PY)
FIELD_TOL_REL = 3e-2        # tests/test_network_gpu.py
# SqueezeNet rounds 26 layers to bf16 in series with nothing that renormalises them (no BatchNorm): the bf16 emulation
# of the seeded nets here is 4-5 % of the field std off at worst (0.6 % on average) where the BatchNorm families stay
# below 1 %
FIELD_TOL_REL_SQUEEZENET = 6e-2


def field_tol(name):
    return FIELD_TOL_REL_SQUEEZENET if name == 'squeezenet' else FIELD_TOL_REL


SHUFFLENETS = ('shufflenetv2x1', 'shufflenetv2x2')


@functools.lru_cache(maxsize=None)
def shell(name, seed=3):
    return tbm.make_pose_shell(name, seed=seed)


@functools.lru_cache(maxsize=None)
def plan(name):
    return network.plan_from_shell(shell(name))


def lowered(p, h, w, **kw):
    tensors, ops, info = network.build_ops(p, h, w, **kw)
    return tensors, [{k: v for k, v in o.items() if not isinstance(v, np.ndarray)} for o in ops], info


@contextlib.contextmanager
def ceil_mode_pools():
    """ops_emulator.run_ops with its max pools in torch's ceil_mode: every pool of a SqueezeNet lowering is one, and
    the interpreter (written for ResNet's floor-mode pool) would give them the floor size"""
    fn = types.SimpleNamespace(**{k: getattr(F, k) for k in dir(F) if not k.startswith('__')})
    fn.max_pool2d = functools.partial(F.max_pool2d, ceil_mode=True)
    with mock.patch.object(ops_emulator, 'F', fn):
        yield


# ---------------------------------------------------------------------------------------------------- the mirror
@pytest.mark.parametrize('size', ['odd', 'even'])
@pytest.mark.parametrize('name', tbm.NAMES)
def test_mirror_equals_stored_reference_module(name, size):
    g = np.load(os.path.join(helpers.GOLDEN_DIR, 'torchvision_backbones.npz'))
    base = tbm.make_pose_shell(name, seed=1).base_net
    with torch.no_grad():
        got = base(torch.from_numpy(g[f'input_{size}']))
    want = torch.from_numpy(g[f'{name}_{size}'])
    assert got.shape == want.shape and got.shape[1] == base.out_features
    torch.testing.assert_close(got, want, rtol=0, atol=1e-5)


def test_stored_features_show_the_ceil_rule():
    """48 x 64 gives SqueezeNet 4 x 5 features (ceil-mode pools: 24 -> 13 -> 7 -> 4); ShuffleNetV2 has 3 x 4"""
    g = np.load(os.path.join(helpers.GOLDEN_DIR, 'torchvision_backbones.npz'))
    assert g['squeezenet_even'].shape[2:] == (4, 5) and g['shufflenetv2x1_even'].shape[2:] == (3, 4)


@pytest.mark.skipif(not HAVE_REF_SRC, reason='reference sources absent')
@pytest.mark.parametrize('name', tbm.NAMES)
def test_mirror_equals_reference_module(name):
    x = torch.randn(1, 3, 42, 58, generator=torch.Generator().manual_seed(5))
    base = tbm.make_pose_shell(name, seed=2).base_net
    with torch.no_grad():
        got = base(x)
    torch.testing.assert_close(got, tbm.reference_features(name, x, base), rtol=0, atol=1e-5)


# ---------------------------------------------------------------------------------------------------- plan and lowering
@pytest.mark.parametrize('h,w', [(67, 83), (96, 64)])
@pytest.mark.parametrize('name,layout', [(n, lay) for n in SHUFFLENETS for lay in ('bins', 'shuffle')] +
                         [('squeezenet', None)])
def test_lowering_reproduces_fp32_and_bf16_emulation(name, layout, h, w):
    x = torch.randn(2, 3, h, w, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = shell(name)(x)
    tensors, ops, _ = network.build_ops(plan(name), h, w, layout=layout)
    with ceil_mode_pools() if name == 'squeezenet' else contextlib.nullcontext():
        got, _ = ops_emulator.run_ops(tensors, ops, x)
        emu, _ = ops_emulator.run_ops(tensors, ops, x, bf16=True)
    assert len(got) == len(want) == 2
    for g, e, wt in zip(got, emu, want):
        assert g.shape == e.shape == wt.shape
        assert float((g - wt).abs().max()) <= 1e-5 * float(wt.abs().max())
        assert float((e - wt).abs().max()) < field_tol(name) * float(wt.std()) + 1e-3
        assert float((e - wt).abs().mean()) < 1e-2 * float(wt.std())


@pytest.mark.parametrize('name', SHUFFLENETS)
def test_shufflenetv2_plan_is_a_shufflenetv2k_plan(name):
    p = plan(name)
    widths = {'shufflenetv2x1': (58, 116, 232, 1024), 'shufflenetv2x2': (122, 244, 488, 2048)}[name]
    assert p['kind'] == 'shufflenetv2k' and 'input2' not in p and 'conv5_stage' not in p
    assert p['input']['w'].shape == (24, 3, 3, 3) and (p['input']['stride'], p['input']['pad']) == (2, 1)
    assert [len(s) for s in p['stages']] == [4, 8, 4]
    for stage, bf in zip(p['stages'], widths):
        assert [b['first'] for b in stage] == [True] + [False] * (len(stage) - 1)
        assert [b['stride'] for b in stage] == [2] + [1] * (len(stage) - 1)
        assert all(b['kernel'] == 3 and b['pad'] == 1 and 'dilation' not in b for b in stage)
        assert all(b['b2_pw2'][0].shape[0] == bf for b in stage)
    assert p['conv5'][0].shape[0] == widths[3] and p['heads'][0]['stride'] == 16


def test_squeezenet_op_list_at_641():
    """stem, 3 ceil-mode pools and 8 Fires (3 conv ops each, the expand pair into one tensor), 41 x 41 features"""
    tensors, ops, info = lowered(plan('squeezenet'), 641, 641)
    assert [o['kind'] for o in ops].count('maxpool') == 3 and [o['kind'] for o in ops].count('conv') == 24
    assert {o['kind'] for o in ops} == {'input_conv', 'maxpool', 'conv', 'heads'}
    assert all(o['ceil_mode'] and o['stride'] == 2 for o in ops if o['kind'] == 'maxpool')
    assert all(o['relu'] == network.ACT_RELU for o in ops if o['kind'] in ('input_conv', 'conv'))
    assert [tensors[o['out']][:2] for o in ops if o['kind'] == 'maxpool'] == [(161, 161), (81, 81), (41, 41)]
    assert tensors[info['feature'][0]] == (41, 41, 512)
    convs = [o for o in ops if o['kind'] == 'conv']
    for sq, e1, e3 in zip(convs[0::3], convs[1::3], convs[2::3]):
        assert sq['kernel'] == e1['kernel'] == 1 and e3['kernel'] == 3 and e3['pad'] == 1
        assert e1['in'] == e3['in'] == sq['out'] and e1['out'] == e3['out']
        assert (e1['out_off'], e3['out_off']) == (0, e1['n_out'])
        assert tensors[e1['out']][2] == network.pad16(e1['n_out'] + e3['n_out'])


@pytest.mark.parametrize('name', tbm.NAMES)
def test_every_tensor_column_is_written_by_one_op(name):
    """the Fire expand pair owns disjoint column windows that cover its output; nothing else writes there"""
    tensors, ops, _ = lowered(plan(name), 97, 130)
    owner = {}
    for i, o in enumerate(ops):
        wins = [(o['out'], 0, network.pad8(o['channels']))] if o['kind'] == 'maxpool' else kr.written_columns(o, tensors)
        for t, c0, c1 in wins:
            assert 0 <= c0 < c1 <= tensors[t][2]
            cols = owner.setdefault(t, np.full(tensors[t][2], -1))
            assert (cols[c0:c1] == -1).all(), (i, t, c0, c1)
            cols[c0:c1] = i
    for o in ops:
        if o['kind'] == 'conv' and o['out_off'] > 0:
            assert (owner[o['out']][:o['out_off'] + o['n_out']] >= 0).all()


# ---------------------------------------------------------------------------------------------------- sizes
@pytest.mark.parametrize('kernel,stride,pad', [(3, 2, 1), (3, 1, 1), (3, 2, 0), (2, 2, 0), (3, 3, 1), (5, 2, 2)])
def test_ceil_mode_size_equals_torch(kernel, stride, pad):
    for n in range(1, 301):
        if n + 2 * pad < kernel:
            continue
        x = torch.empty(1, 1, n, n + 1)
        want = tuple(F.max_pool2d(x, kernel, stride, pad, ceil_mode=True).shape[2:])
        assert network.conv_out_hw(n, n + 1, kernel, stride, pad, ceil_mode=True) == want, n
        want = tuple(F.max_pool2d(x, kernel, stride, pad).shape[2:])
        assert network.conv_out_hw(n, n + 1, kernel, stride, pad) == want, n


CAP = (161, 193)            # tests/test_input_size.py


def sweep():
    """the 41 sizes tests/test_input_size.py sweeps for a stride-16 family"""
    out = ism.sizes(*CAP) + [(15, 13), (1, 1), (CAP[0], 1), (1, CAP[1]), CAP]
    rng = np.random.default_rng(1)
    return out + [(int(rng.integers(1, CAP[0] + 1)), int(rng.integers(1, CAP[1] + 1))) for _ in range(20)]


@pytest.mark.parametrize('name,layout', [(n, lay) for n in SHUFFLENETS for lay in ('bins', 'shuffle')] +
                         [('squeezenet', None)])
def test_tensor_table_equals_lowering_at_each_size(name, layout):
    sizes = sweep()
    assert len(sizes) == 41
    cap_tensors, ops, _ = lowered(plan(name), *CAP, layout=layout)
    for h, w in sizes:
        assert network.tensor_shapes_at(ops, cap_tensors, h, w) == lowered(plan(name), h, w, layout=layout)[0], (h, w)
    with pytest.raises(RuntimeError, match='above its capacity'):
        network.tensor_shapes_at(ops, cap_tensors, CAP[0] + 32, CAP[1])


def test_even_sizes_take_the_ceil_rule():
    """640 -> 320 -> 161 (the floor rule: 160) -> 81 -> 41"""
    tensors, ops, _ = lowered(plan('squeezenet'), 640, 640)
    assert [tensors[o['out']][:2] for o in ops if o['kind'] == 'maxpool'] == [(161, 161), (81, 81), (41, 41)]


# ---------------------------------------------------------------------------------------------------- kernel picks
@pytest.mark.parametrize('name', SHUFFLENETS)
def test_planner_picks_3x3_tma_depthwise_and_no_fused_kernels(name):
    """every depthwise op runs DW_K3_S1 / DW_K3_S2; the stride-2 entry pairs stay two launches (k_pw_dw is the 5x5
    stride-2 kernel) and fuse_dw offers k_dw_gemm nothing (5x5 only)"""
    tensors, ops, _ = lowered(plan(name), 641, 641)
    dws = [o for o in ops if o['kind'] == 'dwconv']
    assert len(dws) == 3 * 2 + 13
    for o in dws:
        assert net_plan.dw_kernel(o['channels'], o['kernel'], o['stride'], o['relu']) == 'DW_K3_S%d' % o['stride']
    assert net_plan.fused_pairs(tensors, ops) == []
    pairs = [(g, d) for g, d in zip(ops, ops[1:]) if g['kind'] == 'conv1x1' and 'pieces' not in g
             and d['kind'] == 'dwconv' and d['in'] == g['out'] and d['stride'] == 2]
    assert len(pairs) == 3
    for g, d in pairs:
        assert net_plan.pw_dw_refusal(g, d, tensors[g['in']][2]) == 'depthwise is not the TMA 5x5 stride-2 kernel'
    assert not any(o['kind'] == 'dw_conv1x1' for o in lowered(plan(name), 641, 641, fuse_dw=True)[1])
    assert all(net_plan.op_cells(o) for o in ops if o['kind'] in ('conv1x1', 'heads'))


def test_squeezenet_convs_take_k_gemm_wg():
    tensors, ops, _ = lowered(plan('squeezenet'), 641, 641)
    routes = [c.route for o in ops for c in net_plan.op_cells(o)]
    assert routes.count('1x1') == 16 and routes.count('conv') == 8 and routes.count('heads') == 1


# ---------------------------------------------------------------------------------------------------- dispatch and refusals
def test_dispatch():
    assert plan('shufflenetv2x1')['kind'] == 'shufflenetv2k' and plan('squeezenet')['kind'] == 'squeezenet'


def refused(name, edit, match):
    s = tbm.make_pose_shell(name, seed=0)
    edit(s.base_net)
    with pytest.raises(network.UnsupportedModel, match=match):
        network.plan_from_shell(s)


def test_other_pool_geometry_is_refused():
    refused('squeezenet', lambda b: setattr(b.backbone[2], 'padding', 0), 'only a 3x3 max pool with padding 1')
    refused('squeezenet', lambda b: setattr(b.backbone[5], 'kernel_size', 2), 'only a 3x3 max pool with padding 1')


def test_fire_without_relu_is_refused():
    refused('squeezenet', lambda b: setattr(b.backbone[3], 'expand3x3_activation', torch.nn.Identity()),
            'expected a ReLU, got Identity')


def test_grouped_conv_is_refused():
    def edit(b):
        b.backbone[4].expand3x3 = torch.nn.Conv2d(16, 64, 3, 1, 1, groups=2)
    refused('squeezenet', edit, 'grouped convolutions')


def test_widths_not_multiples_of_8_are_refused():
    def edit(b):
        fire = b.backbone[12]
        fire.expand1x1 = torch.nn.Conv2d(64, 252, 1)
        fire.expand3x3 = torch.nn.Conv2d(64, 260, 3, 1, 1)
    refused('squeezenet', edit, 'multiples of 8')


def test_expand1x1_width_not_a_multiple_of_16_is_refused():
    """the expand3x3 half of the output starts at column e1, and a conv's output window on a 16-channel boundary"""
    def edit(b):
        fire = b.backbone[12]
        fire.expand1x1 = torch.nn.Conv2d(64, 248, 1)
        fire.expand3x3 = torch.nn.Conv2d(64, 264, 3, 1, 1)
    refused('squeezenet', edit, 'not a multiple of 16')


def test_foreign_module_in_the_squeezenet_backbone_is_refused():
    refused('squeezenet', lambda b: b.backbone.__setitem__(6, torch.nn.Identity()), 'a MaxPool2d or a Fire module')


def test_shufflenetv2_conv5_without_relu_is_refused():
    refused('shufflenetv2x1', lambda b: b.conv5.__setitem__(2, torch.nn.Identity()), 'conv5: expected Conv2d')


def test_mobilenetv3_large_is_still_refused_with_hardswish():
    import torchvision
    import mobilenetv2_models as mm
    base = mm.MobileNetV2('mobilenetv3large', 960)
    base.backbone = list(torchvision.models.mobilenet_v3_large(weights=None).children())[0]
    with pytest.raises(network.UnsupportedModel, match='Hardswish'):
        network.plan_from_shell(mm.make_pose_shell(seed=0, base=base))
