"""Test infrastructure: fp32 PyTorch restatement of the reference's MobileNetV2 base network and counters of the op list
openpifpaf_b200.network.build_ops emits for it (paths relative to the reference's src/openpifpaf/):

  MobileNetV2          network/basenetworks.py:407-417 (backbone = torchvision mobilenet_v2().features, stride 32)

The module attribute names and state_dict keys equal the reference's, so its own module loads these weights
unchanged (tests/test_mobilenetv2.py compares the two).  Torchvision is always asked for weights=None."""
import torch

import det_models
from openpifpaf_b200 import constants
from oracle import net_oracle


class MobileNetV2(torch.nn.Module):
    """basenetworks.py:407-417: the features of torchvision's mobilenet_v2, the classifier removed."""

    def __init__(self, name='mobilenetv2', out_features=1280, **tv_kwargs):
        super().__init__()
        import torchvision
        self.name, self.stride, self.out_features = name, 32, out_features
        self.backbone = list(torchvision.models.mobilenet_v2(weights=None, **tv_kwargs).children())[0]

    def forward(self, x):
        return self.backbone(x)


def make_pose_shell(seed=0, base=None):
    """MobileNetV2 + the CocoKp heads (Cif 17, Caf 19 with the COCO person skeleton), seeded as det_models.seed_shell
    seeds (random BatchNorm statistics, eval mode)."""
    base = MobileNetV2() if base is None else base
    cif, caf = net_oracle.HeadMeta.cif(17), net_oracle.HeadMeta.caf(19)
    caf.skeleton = constants.COCO_PERSON_SKELETON
    heads = [net_oracle.CompositeField4(cif, base.out_features), net_oracle.CompositeField4(caf, base.out_features)]
    return det_models.seed_shell(net_oracle.Shell(base, heads), seed)


def calibrate_pose_heads(shell, confidence_bias=-1.75, size=161):
    """Centre and rescale every head channel on the features of a probe batch (as network.calibrate_random_heads does
    for plans) and shift the confidences, so that a from-scratch net emits isolated confident cells that decode into
    some poses instead of a saturated map."""
    dev = next(shell.parameters()).device
    with torch.no_grad():
        feat = shell.base_net(torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(7)).to(dev))
        mu = feat.mean((0, 2, 3))
        for hn in shell.head_nets:
            w = hn.conv.weight[:, :, 0, 0]
            pre = torch.einsum('nc,bchw->bnhw', w, feat - mu[None, :, None, None])
            w = w / pre.std((0, 2, 3))[:, None]
            hn.conv.bias.copy_(-(w @ mu))
            hn.conv.weight.copy_(w[:, :, None, None])
            hn.conv.bias.view(hn.meta.n_fields, -1)[:, 1] += confidence_bias
    return shell


def reference_features(x, oracle_base):
    """The reference's own basenetworks.MobileNetV2 (pretrained off) loaded with the weights of `oracle_base`, applied
    to x.  Needs the reference sources."""
    import torchvision
    from oracle import make_golden
    _, base, _ = make_golden.load_reference_modules()
    saved = base.MobileNetV2.pretrained
    try:
        base.MobileNetV2.pretrained = False
        ref = base.MobileNetV2('mobilenetv2', lambda pretrained: torchvision.models.mobilenet_v2(weights=None))
    finally:
        base.MobileNetV2.pretrained = saved
    assert ref.stride == oracle_base.stride == 32 and ref.out_features == oracle_base.out_features
    ref.load_state_dict(oracle_base.state_dict())
    net_oracle.model_defaults(ref)
    ref.eval()
    with torch.no_grad():
        return ref(x)


def golden_input():
    return torch.randn(1, 3, 49, 65, generator=torch.Generator().manual_seed(23))


def op_counts(ops):
    """(convolutions, depthwise convolutions, residual adds) of a MobileNetV2 op list, the heads not counted"""
    convs = [o for o in ops if o['kind'] in ('input_conv', 'conv', 'dwconv')]
    return (len(convs), sum(o['kind'] == 'dwconv' for o in ops),
            sum(o['kind'] == 'conv' and o['residual'] >= 0 for o in ops))


def algorithmic_bytes(tensors, ops, batch=1):
    """bf16 bytes of the input and output of every conv (real channels, images as f32), per op kind"""
    out = {}
    for o in ops:
        k = o['kind']
        if k == 'input_conv':
            h, w, _ = tensors[o['out']]
            n = o['in_h'] * o['in_w'] * 3 * 4 + h * w * o['c_out'] * 2
        elif k in ('conv', 'dwconv'):
            c_in = o['c_in'] if k == 'conv' else o['channels']
            c_out = o['n_out'] if k == 'conv' else o['channels']
            hi, wi, _ = tensors[o['in']]
            ho, wo, _ = tensors[o['out']]
            n = hi * wi * c_in * 2 + ho * wo * c_out * 2 * (2 if k == 'conv' and o['residual'] >= 0 else 1)
            if k == 'conv':
                k = 'conv residual' if o['residual'] >= 0 else 'conv'
        else:
            continue
        out[k] = out.get(k, 0) + n * batch
    return out


def flops(tensors, ops):
    """multiply-adds x 2 of the convolutions of one image"""
    total = 0
    for o in ops:
        if o['kind'] == 'input_conv':
            h, w, _ = tensors[o['out']]
            total += 2 * h * w * o['c_out'] * 3 * o['kernel'] ** 2
        elif o['kind'] == 'conv':
            h, w, _ = tensors[o['out']]
            total += 2 * h * w * o['n_out'] * o['c_in'] * o['kernel'] ** 2
        elif o['kind'] == 'dwconv':
            h, w, _ = tensors[o['out']]
            total += 2 * h * w * o['channels'] * o['kernel'] ** 2
    return total
