"""CPU: the per-size tensor table `CompiledNet.set_input_size` hands to the library equals the lowering at that size,
for every plan family, and sizes above the capacity or that empty a layer are refused."""
import numpy as np
import pytest

import input_size_models as ism
from openpifpaf_b200 import network

CAP = (161, 193)


def lowered(name, h, w, **kw):
    tensors, ops, _ = network.build_ops(ism.plan(name), h, w, **kw)
    return tensors, [{k: v for k, v in o.items() if not isinstance(v, np.ndarray)} for o in ops]


def sweep(name):
    cap = CAP
    out = ism.sizes(*cap) + [ism.tiny(name), (1, 1), (cap[0], 1), (1, cap[1]), cap]
    rng = np.random.default_rng(1)
    out += [(int(rng.integers(1, cap[0] + 1)), int(rng.integers(1, cap[1] + 1))) for _ in range(20)]
    return out


def test_sizes_cover_every_residue_and_both_orientations():
    s = ism.sizes(*CAP)
    assert {h % 16 for h, _ in s} == set(range(16)) and {w % 16 for _, w in s} == set(range(16))
    assert any(h > w for h, w in s) and any(h < w for h, w in s)
    assert all(1 <= h <= CAP[0] and 1 <= w <= CAP[1] for h, w in s)


@pytest.mark.parametrize('name', sorted(ism.FAMILIES))
def test_tensor_table_equals_lowering_at_each_size(name):
    cap_tensors, ops = lowered(name, *CAP)
    for h, w in sweep(name):
        assert network.tensor_shapes_at(ops, cap_tensors, h, w) == lowered(name, h, w)[0], (h, w)


@pytest.mark.parametrize('kw', [dict(layout='shuffle'), dict(fuse_dw=True)], ids=['shuffle', 'fuse_dw'])
def test_tensor_table_of_other_shufflenet_lowerings(kw):
    cap_tensors, ops = lowered('k16', *CAP, **kw)
    assert any(o['kind'] == 'dw_conv1x1' for o in ops) == ('fuse_dw' in kw)
    for h, w in sweep('k16'):
        assert network.tensor_shapes_at(ops, cap_tensors, h, w) == lowered('k16', h, w, **kw)[0], (h, w)


@pytest.mark.parametrize('name', sorted(ism.FAMILIES))
def test_tiny_size_gives_one_cell_fields(name):
    tensors, ops = lowered(name, *ism.tiny(name))
    feat = ops[-1]['in']
    assert tensors[feat][:2] == (1, 1)      # and the heads' crop of an upsampled 1 x 1 map keeps one cell


@pytest.mark.parametrize('name', sorted(ism.FAMILIES))
def test_sizes_above_capacity_are_refused(name):
    cap_tensors, ops = lowered(name, *CAP)
    # one more input pixel may round to the same tensors (the stem's stride); 32 more never does
    for h, w in [(CAP[0] + 32, CAP[1]), (CAP[0], CAP[1] + 32), (CAP[1], CAP[0])]:
        with pytest.raises(RuntimeError, match='above its capacity'):
            network.tensor_shapes_at(ops, cap_tensors, h, w)


def test_sizes_that_empty_a_layer_are_refused():
    """a 7x7 stem without padding has no output below 7 pixels"""
    plan = network.random_resnet_plan('resnet18', seed=0)
    plan['input']['pad'] = 0
    cap_tensors, ops, _ = network.build_ops(plan, *CAP)
    ops = [{k: v for k, v in o.items() if not isinstance(v, np.ndarray)} for o in ops]
    assert network.tensor_shapes_at(ops, cap_tensors, 7, 7)[0][:2] == (1, 1)
    for h, w in [(6, 100), (100, 6), (1, 1)]:
        with pytest.raises(RuntimeError, match='empty output'):
            network.tensor_shapes_at(ops, cap_tensors, h, w)
