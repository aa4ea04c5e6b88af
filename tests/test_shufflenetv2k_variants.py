"""CPU: the structural options of the reference's ShuffleNetV2K (basenetworks.py:245-405:
--shufflenetv2k-stage4-dilation, --shufflenetv2k-input-conv2-stride / -outchannels, --shufflenetv2k-conv5-as-stage).
(1) The test mirror in shufflenetv2k_models.py equals the reference's own modules (stored features, and the live
modules where the reference sources exist); (2) the product's lowering reproduces it in both activation layouts when
its op list runs in the CPU interpreter; (3) random_plan builds the geometry plan_from_shell extracts; (4) the
default plan is unchanged and the layer options the compiled forward cannot serve are still refused."""
import os

import numpy as np
import pytest
import torch

import helpers
import ops_emulator
import shufflenetv2k_models as sm
from openpifpaf_b200 import network
from oracle import build_ref, net_oracle

HAVE_REF_SRC = os.path.isdir(build_ref.REF_PY)
CASES = [(v, 'tiny') for v in sm.VARIANTS] + [('conv5stage', 'tiny_wide')]


def case_id(c):
    return '%s-%s' % c


@pytest.mark.parametrize('variant,config', CASES, ids=[case_id(c) for c in CASES])
def test_variant_equals_stored_reference_module(variant, config):
    g = np.load(os.path.join(helpers.GOLDEN_DIR, 'shufflenetv2k_variants.npz'))
    base = sm.make_pose_shell(variant, config, seed=1).base_net
    with torch.no_grad():
        got = base(torch.from_numpy(g['input']))
    want = torch.from_numpy(g[f'{variant}/{config}'])
    assert got.shape == want.shape
    torch.testing.assert_close(got, want, rtol=0, atol=1e-5)


@pytest.mark.skipif(not HAVE_REF_SRC, reason='reference sources absent')
@pytest.mark.parametrize('variant,config', CASES, ids=[case_id(c) for c in CASES])
def test_variant_equals_reference_module(variant, config):
    x = torch.randn(1, 3, 53, 67, generator=torch.Generator().manual_seed(5))
    base = sm.make_pose_shell(variant, config, seed=2).base_net
    with torch.no_grad():
        got = base(x)
    torch.testing.assert_close(got, sm.reference_features(variant, x, base), rtol=0, atol=1e-5)


def test_mirror_defaults_equal_the_oracle():
    """without options the mirror is net_oracle.ShuffleNetV2K: same state_dict keys and shapes, same features"""
    repeats, channels = sm.CONFIGS['tiny']
    mine = sm.ShuffleNetV2K('tiny', repeats, channels)
    theirs = net_oracle.ShuffleNetV2K('tiny', repeats, channels)
    assert {k: v.shape for k, v in mine.state_dict().items()} == {k: v.shape for k, v in theirs.state_dict().items()}
    theirs.load_state_dict(mine.state_dict())
    mine.eval()
    theirs.eval()
    x = torch.randn(1, 3, 37, 45, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        torch.testing.assert_close(mine(x), theirs(x), rtol=0, atol=0)


@pytest.mark.parametrize('layout', ['bins', 'shuffle'])
@pytest.mark.parametrize('variant,config', CASES, ids=[case_id(c) for c in CASES])
def test_variant_lowering_reproduces_mirror(variant, config, layout):
    shell = sm.make_pose_shell(variant, config, seed=3)
    h, w = 77, 93
    x = torch.randn(2, 3, h, w, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = shell(x)
    plan = network.plan_from_shell(shell)
    tensors, ops, info = network.build_ops(plan, h, w, layout=layout)
    got, acts = ops_emulator.run_ops(tensors, ops, x)
    assert len(got) == len(want)
    for g, wt in zip(got, want):
        assert g.shape == wt.shape
        assert float((g - wt).abs().max()) <= 1e-5 * float(wt.abs().max())
    # the feature tensor and its layout are what the heads read
    t, lay = info['feature']
    with torch.no_grad():
        feat = shell.base_net(x).permute(0, 2, 3, 1)
    got_feat = acts[t][..., lay.cols()]
    assert float((got_feat - feat).abs().max()) <= 1e-5 * float(feat.abs().max())
    opts = sm.VARIANTS[variant]
    dil = opts.get('stage4_dilation', 1)
    assert {o.get('dilation', 1) for o in ops if o['kind'] == 'dwconv'} == ({1, dil} if dil > 1 else {1})
    assert sum(o['kind'] == 'conv' for o in ops) == (1 if opts.get('input_conv2_stride') else 0)
    for hd, hn in zip(plan['heads'], shell.head_nets):
        assert hd['stride'] == shell.base_net.stride // hn.meta.upsample_stride == hn.meta.stride


def test_dilated_head_stride_is_8():
    shell = sm.make_pose_shell('dil2', 'tiny')
    plan = network.plan_from_shell(shell)
    assert shell.base_net.stride == 8 and all(hd['stride'] == 8 for hd in plan['heads'])
    tensors, ops, _ = network.build_ops(plan, 641, 641)
    assert tensors[ops[-1]['in']][:2] == (81, 81)


def test_dilated_ops_are_never_fused():
    """fuse_dw only takes the undilated 5x5: a dilated depthwise op stays a dwconv op"""
    plan = network.random_plan('shufflenetv2k16', stage4_dilation=2, conv5_as_stage=True)
    _, ops, _ = network.build_ops(plan, 161, 161, fuse_dw=True)
    assert all(o.get('dilation', 1) == 1 for o in ops if o['kind'] == 'dw_conv1x1')
    assert sum(o.get('dilation', 1) == 2 for o in ops if o['kind'] == 'dwconv') == 4 + 1 + 2


RANDOM_OPTS = {
    'dil2': dict(stage4_dilation=2),
    'conv2': dict(input_conv2_stride=2),
    'conv2_out48': dict(input_conv2_stride=2, input_conv2_outchannels=48),
    'conv5stage': dict(conv5_as_stage=True),
    'dil2_conv5stage': dict(stage4_dilation=2, conv5_as_stage=True),
    'conv2_dil2': dict(input_conv2_stride=2, stage4_dilation=2),
}


def geometry(p):
    def block(e):
        return (e['first'], e['stride'], e['kernel'], e['pad'], e.get('dilation', 1),
                tuple(tuple(e[k][0].shape) for k in ('b2_pw1', 'b2_dw', 'b2_pw2', 'b1_dw', 'b1_pw') if k in e))
    return (p['input']['w'].shape, p['input']['stride'], p['input']['pad'],
            None if 'input2' not in p else (p['input2']['w'].shape, p['input2']['stride'], p['input2']['pad']),
            [[block(e) for e in s] for s in p['stages']],
            None if 'conv5' not in p else p['conv5'][0].shape,
            None if 'conv5_stage' not in p else [block(e) for e in p['conv5_stage']],
            [(h['w'].shape, h['stride'], h['ops']) for h in p['heads']])


@pytest.mark.parametrize('variant', list(RANDOM_OPTS))
def test_random_plan_matches_extracted_plan(variant):
    """random_plan(**options) has the architecture plan_from_shell extracts from the same ShuffleNetV2K variant"""
    repeats, channels = net_oracle.SHUFFLENETV2K_CONFIGS['shufflenetv2k16']
    base = sm.ShuffleNetV2K('shufflenetv2k16', repeats, channels, **sm.VARIANTS[variant])
    heads = [net_oracle.CompositeField4(net_oracle.HeadMeta.cif(17), base.out_features),
             net_oracle.CompositeField4(net_oracle.HeadMeta.caf(19), base.out_features)]
    shell = net_oracle.Shell(base, heads).eval()
    want = network.plan_from_shell(shell)
    got = network.random_plan('shufflenetv2k16', **RANDOM_OPTS[variant])
    assert geometry(got) == geometry(want)


def test_random_plan_conv5_stage_with_branch1():
    """a conv5 wider than stage 4: the first conv5-as-stage block has a branch1, as the reference builds it"""
    base = sm.make_base('conv5stage', 'tiny_wide')
    assert base.conv5[0].branch1 is not None
    plan = network.plan_from_shell(sm.make_pose_shell('conv5stage', 'tiny_wide'))
    assert [e['first'] for e in plan['conv5_stage']] == [True, False]
    assert plan['conv5_stage'][0]['stride'] == 1


def test_default_plan_is_unchanged():
    """the new plan keys are additive: the default plan has no 'input2' / 'conv5_stage' and no 'dilation'"""
    for plan in (network.plan_from_shell(net_oracle.make_shell('shufflenetv2k16', seed=0)),
                 network.random_plan('shufflenetv2k16')):
        assert 'input2' not in plan and 'conv5_stage' not in plan and 'conv5' in plan
        assert all('dilation' not in e for s in plan['stages'] for e in s)
        assert all(hd['stride'] == 16 for hd in plan['heads'])


def _with_module(shell, path, make):
    parent = shell.base_net
    for p in path[:-1]:
        parent = getattr(parent, p) if not p.isdigit() else parent[int(p)]
    parent[int(path[-1])] = make()
    return shell


def test_leaky_relu_is_refused():
    shell = _with_module(sm.make_pose_shell('dil2', 'tiny'), ['stage4', '0', 'branch2', '2'],
                         lambda: torch.nn.LeakyReLU(inplace=True))
    with pytest.raises(network.UnsupportedModel, match='LeakyReLU'):
        network.plan_from_shell(shell)


def test_group_norm_is_refused():
    shell = _with_module(sm.make_pose_shell('conv5stage', 'tiny'), ['conv5', '0', 'branch2', '1'],
                         lambda: torch.nn.GroupNorm(4, 32))
    with pytest.raises(network.UnsupportedModel, match='GroupNorm'):
        network.plan_from_shell(shell)
