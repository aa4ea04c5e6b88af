"""CPU: the Resnet options of the reference's constructor and CLI (basenetworks.py:71-150: --resnet-pool0-stride,
--resnet-input-conv-stride, --resnet-input-conv2-stride, --resnet-block5-dilation) and the resnet18-cocodet recipe
with its upsample-2 CifDet head.  (1) The test mirror in det_models.py equals the reference's own modules (stored
features, and the live modules where the reference sources exist); (2) the product's lowering reproduces it when
its op list runs in the CPU interpreter; (3) the two options the compiled forward cannot serve are refused."""
import os

import numpy as np
import pytest
import torch

import det_models
import helpers
import ops_emulator
from openpifpaf_b200 import network
from oracle import build_ref, net_oracle

HAVE_REF_SRC = os.path.isdir(build_ref.REF_PY)
VARIANTS = list(det_models.VARIANTS)


@pytest.mark.parametrize('variant', VARIANTS)
def test_variant_equals_stored_reference_module(variant):
    g = np.load(os.path.join(helpers.GOLDEN_DIR, 'resnet_variants.npz'))
    base = det_models.make_variant_shell(variant, seed=1).base_net
    with torch.no_grad():
        got = base(torch.from_numpy(g['input']))
    want = torch.from_numpy(g[variant])
    assert got.shape == want.shape
    torch.testing.assert_close(got, want, rtol=0, atol=1e-5)


@pytest.mark.skipif(not HAVE_REF_SRC, reason='reference sources absent')
@pytest.mark.parametrize('variant', VARIANTS)
def test_variant_equals_reference_module(variant):
    x = torch.randn(1, 3, 41, 57, generator=torch.Generator().manual_seed(5))
    base = det_models.make_variant_shell(variant, seed=2).base_net
    with torch.no_grad():
        got = base(x)
    torch.testing.assert_close(got, det_models.reference_resnet_features(variant, x, base), rtol=0, atol=1e-5)


# every variant on resnet18; the Bottleneck blocks of resnet50 with the max pool, dilation and the cocodet recipe
@pytest.mark.parametrize('variant,base_name', [(v, 'resnet18') for v in VARIANTS] +
                         [(v, 'resnet50') for v in ('pool2', 'dil2', 'cocodet')])
def test_variant_lowering_reproduces_oracle(variant, base_name):
    shell = det_models.make_variant_shell(variant, base_name=base_name, seed=3)
    h, w = 53, 71
    x = torch.randn(2, 3, h, w, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = shell(x)
    plan = network.plan_from_shell(shell)
    tensors, ops, _ = network.build_ops(plan, h, w)
    got, _ = ops_emulator.run_ops(tensors, ops, x)
    assert len(got) == len(want)
    for g, wt in zip(got, want):
        assert g.shape == wt.shape
        assert float((g - wt).abs().max()) <= 1e-5 * float(wt.abs().max())
    kinds = [o['kind'] for o in ops]
    opts = det_models.VARIANTS[variant]
    assert ('maxpool' in kinds) == bool(opts.get('pool0_stride'))
    dil = opts.get('block5_dilation', 1)
    assert {o['dilation'] for o in ops if o['kind'] == 'conv' and o['kernel'] > 1} == ({1, dil} if dil > 1 else {1})
    # the plan's head stride is the reference's: base.stride // upsample_stride (heads.py, headmeta.stride)
    for hd, hn in zip(plan['heads'], shell.head_nets):
        assert hd['stride'] == shell.base_net.stride // hn.meta.upsample_stride == hn.meta.stride


def test_default_plan_is_unchanged():
    """the new plan keys are additive: the default Resnet plan has no 'pool' / 'input2' and no conv 'dilation'"""
    plan = network.plan_from_shell(net_oracle.make_shell('resnet18', seed=0))
    assert 'pool' not in plan and 'input2' not in plan
    assert all('dilation' not in c for b in plan['blocks'] for c in b['convs'] + [b['downsample'] or {}])


@pytest.mark.parametrize('variant', ['pool2', 'pool1', 'stem_s1', 'conv2', 'dil2', 'cocodet'])
def test_random_resnet_plan_matches_extracted_plan(variant):
    """random_resnet_plan(**options) has the architecture plan_from_shell extracts from the same Resnet variant"""
    opts = dict(det_models.VARIANTS[variant])
    shell = det_models.make_variant_shell(variant, seed=0)
    want = network.plan_from_shell(shell)
    up = shell.head_nets[0].meta.upsample_stride
    heads = ((91, 1, 2, 0, (True, False)),) if variant == 'cocodet' else ((17, 1, 1, 1), (19, 1, 2, 2))
    got = network.random_resnet_plan('resnet18', heads=heads, upsample=up, **opts)

    def geometry(p):
        convs = [p['input']] + ([p['input2']] if 'input2' in p else [])
        convs += [c for b in p['blocks'] for c in b['convs'] + ([b['downsample']] if b['downsample'] else [])]
        return ([(c['w'].shape, c['stride'], c['pad'], c.get('dilation', 1)) for c in convs], p.get('pool'),
                [(h['w'].shape, h['stride'], h.get('upsample', 1), h['ops']) for h in p['heads']])
    assert geometry(got) == geometry(want)


def test_grouped_convolutions_are_refused():
    import torchvision
    base = det_models.Resnet('resnext50', lambda weights: torchvision.models.resnext50_32x4d(weights=weights), 2048)
    shell = det_models.make_det_shell(base, 3, 1)
    with pytest.raises(RuntimeError, match='grouped'):
        network.plan_from_shell(shell)


def test_remove_last_block_is_refused():
    base = det_models.make_resnet('resnet18', remove_last_block=True)
    shell = det_models.make_det_shell(base, 3, 1)
    with pytest.raises(RuntimeError, match='remove_last_block'):
        network.plan_from_shell(shell)


def test_unsupported_pool_is_refused():
    base = det_models.make_resnet('resnet18', pool0_stride=2)
    base.input_block[3].kernel_size = 2
    with pytest.raises(RuntimeError, match='max pool'):
        network.plan_from_shell(det_models.make_det_shell(base, 3, 1))
