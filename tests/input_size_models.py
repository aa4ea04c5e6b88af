"""Plans of every family the compiled forward lowers, and the input sizes the variable-size tests run them at.

A net is compiled at a capacity and run at smaller sizes (`network.CompiledNet.set_input_size`).  `sizes(cap_h, cap_w)`
gives sizes below a capacity that cover every residue mod 16 in both dimensions (so each stride-2 layer rounds both
ways), both orientations and odd sizes; `tiny(name)` is a size whose head fields are 1 x 1."""
import functools

import numpy as np

from openpifpaf_b200 import network

CIFDET_HEADS = ((91, 1, 2, 0, (True, False)),)

FAMILIES = {
    'k16': lambda: network.random_plan('shufflenetv2k16', seed=1),
    'k16_dil2': lambda: network.random_plan('shufflenetv2k16', seed=2, stage4_dilation=2),
    'k16_conv2': lambda: network.random_plan('shufflenetv2k16', seed=3, input_conv2_stride=2),
    'k16_conv5stage': lambda: network.random_plan('shufflenetv2k16', seed=4, conv5_as_stage=True),
    'resnet50_pool': lambda: network.random_resnet_plan('resnet50', seed=5, pool0_stride=2),
    'resnet18_conv2_dil2': lambda: network.random_resnet_plan('resnet18', seed=6, input_conv2_stride=2,
                                                              block5_dilation=2),
    'cifdet_up2': lambda: network.random_resnet_plan('resnet18', heads=CIFDET_HEADS, seed=7, input_conv2_stride=2,
                                                     block5_dilation=2, upsample=2),
    'mobilenetv2': lambda: _mobilenetv2_plan(),
    'heads_only': lambda: network.heads_only_plan(network.random_plan('shufflenetv2k16', seed=8)),
}


def _mobilenetv2_plan():
    import mobilenetv2_models
    return network.plan_from_shell(mobilenetv2_models.make_pose_shell(seed=9))


@functools.lru_cache(maxsize=None)
def plan(name):
    return FAMILIES[name]()


def input_stride(name):
    """input pixels per feature cell (1 for a heads-only plan, whose input is the feature map)"""
    p = plan(name)
    if p['kind'] == 'heads_only':
        return 1
    hd = p['heads'][0]
    return hd['stride'] * hd.get('upsample', 1)


def tiny(name):
    """an odd size, both sides below the feature stride: every feature map, and so every head field, is 1 x 1"""
    s = input_stride(name)
    return (max(1, s - 1), max(1, s - 3))


def sizes(cap_h, cap_w, seed=0):
    """16 sizes (h, w) <= (cap_h, cap_w), one per residue r: h % 16 == r and w % 16 == 15 - r, drawn from a seeded
    generator; sizes alternate between landscape and portrait where the capacity allows it"""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(16):
        for _ in range(100):
            h = int(rng.integers(0, (cap_h - r) // 16 + 1)) * 16 + r
            w = int(rng.integers(0, (cap_w - 15 + r) // 16 + 1)) * 16 + 15 - r
            if h >= 1 and w >= 1 and (h > w) == (r % 2 == 0) and (h, w) != (cap_h, cap_w):
                break
        out.append((h, w))
    return out
