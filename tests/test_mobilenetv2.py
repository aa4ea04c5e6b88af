"""CPU: the MobileNetV2 base network of the reference (basenetworks.py:407-417).  (1) The test mirror in
mobilenetv2_models.py equals the reference's own module (stored features, and the live module where the reference
sources exist); (2) the product's lowering reproduces the fp32 Shell when its op list runs in the CPU interpreter, and
stays within the field tolerance in the bf16 emulation; (3) MobileNetV3 and MobileNetV2 variants the compiled forward
does not implement are refused."""
import os

import numpy as np
import pytest
import torch

import helpers
import mobilenetv2_models as mm
import ops_emulator
from openpifpaf_b200 import network
from oracle import build_ref, net_oracle

HAVE_REF_SRC = os.path.isdir(build_ref.REF_PY)
FIELD_TOL_REL = 3e-2        # tests/test_network_gpu.py


def test_mirror_equals_stored_reference_module():
    g = np.load(os.path.join(helpers.GOLDEN_DIR, 'mobilenetv2.npz'))
    base = mm.make_pose_shell(seed=1).base_net
    with torch.no_grad():
        got = base(torch.from_numpy(g['input']))
    want = torch.from_numpy(g['features'])
    assert got.shape == want.shape == (1, 1280, 2, 3)
    torch.testing.assert_close(got, want, rtol=0, atol=1e-5)


@pytest.mark.skipif(not HAVE_REF_SRC, reason='reference sources absent')
def test_mirror_equals_reference_module():
    x = torch.randn(1, 3, 41, 57, generator=torch.Generator().manual_seed(5))
    base = mm.make_pose_shell(seed=2).base_net
    with torch.no_grad():
        got = base(x)
    torch.testing.assert_close(got, mm.reference_features(x, base), rtol=0, atol=1e-5)


@pytest.mark.parametrize('h,w', [(67, 83), (97, 65)])
def test_lowering_reproduces_fp32_and_bf16_emulation(h, w):
    shell = mm.make_pose_shell(seed=3)
    x = torch.randn(2, 3, h, w, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = shell(x)
    plan = network.plan_from_shell(shell)
    tensors, ops, _ = network.build_ops(plan, h, w)
    got, _ = ops_emulator.run_ops(tensors, ops, x)
    emu, _ = ops_emulator.run_ops(tensors, ops, x, bf16=True)
    assert len(got) == len(want) == 2
    for g, e, wt in zip(got, emu, want):
        assert g.shape == e.shape == wt.shape
        assert float((g - wt).abs().max()) <= 1e-5 * float(wt.abs().max())
        assert float((e - wt).abs().max()) < FIELD_TOL_REL * float(wt.std()) + 1e-3


def test_op_list_at_641():
    """52 convolutions (17 depthwise), 10 residual adds in the projection epilogue, ReLU6 everywhere but the
    projections, 5.1 GFLOP per image, 21 x 21 heads"""
    plan = network.plan_from_shell(mm.make_pose_shell(seed=0))
    tensors, ops, info = network.build_ops(plan, 641, 641)
    assert mm.op_counts(ops) == (52, 17, 10)
    assert {o['kind'] for o in ops} == {'input_conv', 'conv', 'dwconv', 'heads'}
    assert all(o['kernel'] == 3 and o['relu'] == network.ACT_RELU6 for o in ops if o['kind'] == 'dwconv')
    projections = [o for o in ops if o['kind'] == 'conv' and o['relu'] == network.ACT_NONE]
    assert len(projections) == 17 and all(o['kernel'] == 1 for o in projections)
    assert all(o['relu'] == network.ACT_RELU6 for o in ops if o['kind'] in ('input_conv', 'conv') and o not in projections)
    assert 5.1e9 < mm.flops(tensors, ops) < 5.2e9
    assert tensors[info['feature'][0]] == (21, 21, 1280)
    assert all(c % 16 == 0 for _, _, c in tensors)
    assert plan['heads'][0]['stride'] == 32
    # block 1 has no expand conv; 24 channels are padded to 32
    assert plan['blocks'][0]['expand'] is None and all(b['expand'] is not None for b in plan['blocks'][1:])
    assert tensors[ops[5]['out']] == (161, 161, 32) and ops[5]['n_out'] == 24


def test_mobilenetv3_small_is_refused():
    import torchvision
    base = mm.MobileNetV2('mobilenetv3small', 576)
    base.backbone = list(torchvision.models.mobilenet_v3_small(weights=None).children())[0]
    shell = mm.make_pose_shell(seed=0, base=base)
    with pytest.raises(network.UnsupportedModel, match='Hardswish'):
        network.plan_from_shell(shell)


def test_hardswish_in_a_v2_block_is_refused():
    shell = mm.make_pose_shell(seed=0)
    shell.base_net.backbone[5].conv[1][2] = torch.nn.Hardswish()
    with pytest.raises(network.UnsupportedModel, match='Hardswish'):
        network.plan_from_shell(shell)


def test_relu_in_place_of_relu6_is_refused():
    shell = mm.make_pose_shell(seed=0)
    shell.base_net.backbone[7].conv[0][2] = torch.nn.ReLU()
    with pytest.raises(network.UnsupportedModel, match='only ReLU6'):
        network.plan_from_shell(shell)


def test_other_width_rounding_is_refused():
    """width_mult 0.75 rounded to multiples of 4 gives 12-channel layers"""
    shell = mm.make_pose_shell(seed=0, base=mm.MobileNetV2(width_mult=0.75, round_nearest=4))
    with pytest.raises(network.UnsupportedModel, match='multiples of 8'):
        network.plan_from_shell(shell)


def test_foreign_module_in_the_backbone_is_refused():
    shell = mm.make_pose_shell(seed=0)
    shell.base_net.backbone[3] = torch.nn.Identity()
    with pytest.raises(network.UnsupportedModel, match='InvertedResidual'):
        network.plan_from_shell(shell)


def test_resnet_and_shufflenet_plans_are_unchanged_by_the_backbone_dispatch():
    assert network.plan_from_shell(net_oracle.make_shell('resnet18', seed=0))['kind'] == 'resnet'
    assert network.plan_from_shell(net_oracle.make_shell('shufflenetv2k16', seed=0))['kind'] == 'shufflenetv2k'
