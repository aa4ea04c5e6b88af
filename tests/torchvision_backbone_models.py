"""Test infrastructure: fp32 PyTorch restatement of the reference's torchvision-backed ShuffleNetV2 and SqueezeNet base
networks (paths relative to the reference's src/openpifpaf/):

  ShuffleNetV2   network/basenetworks.py:36-68   (torchvision shufflenet_v2_x1_0 / x2_0 without the max pool, stride 16)
  SqueezeNet     network/basenetworks.py:461-499 (torchvision squeezenet1_1().features with every max pool padded by 1
                                                  and every conv padded by (k - 1) // 2, stride 16)

The module attribute names and state_dict keys equal the reference's, so its own modules load these weights unchanged
(tests/test_torchvision_backbones.py compares the two).  Torchvision is always asked for weights=None."""
import torch

import det_models
from openpifpaf_b200 import constants
from oracle import net_oracle

SHUFFLENETV2 = {          # network/factory.py: name -> (torchvision constructor, out_features)
    'shufflenetv2x1': ('shufflenet_v2_x1_0', 1024),
    'shufflenetv2x2': ('shufflenet_v2_x2_0', 2048),
}
NAMES = tuple(SHUFFLENETV2) + ('squeezenet',)


class ShuffleNetV2(torch.nn.Module):
    """basenetworks.py:36-68: conv1, stage2..4 and conv5 of torchvision's ShuffleNetV2; its max pool is not used."""

    def __init__(self, name='shufflenetv2x1'):
        super().__init__()
        import torchvision
        ctor, out_features = SHUFFLENETV2[name]
        tv = getattr(torchvision.models, ctor)(weights=None)
        self.name, self.stride, self.out_features = name, 16, out_features
        self.conv1, self.stage2, self.stage3, self.stage4, self.conv5 = tv.conv1, tv.stage2, tv.stage3, tv.stage4, tv.conv5

    def forward(self, x):
        return self.conv5(self.stage4(self.stage3(self.stage2(self.conv1(x)))))


def squeezenet_padding(module):
    """The reference's edits of torchvision's SqueezeNet: a max pool whose padding is not 1 gets 1 (the ceil_mode
    pools stay ceil_mode), a conv whose padding is not (k - 1) // 2 gets it (the stem: 0 -> 1)."""
    for m in module.modules():
        if isinstance(m, torch.nn.MaxPool2d) and m.padding != 1:
            m.padding = 1
        if isinstance(m, torch.nn.Conv2d) and m.padding[0] != (m.kernel_size[0] - 1) // 2:
            m.padding = ((m.kernel_size[0] - 1) // 2,) * 2
    return module


class SqueezeNet(torch.nn.Module):
    """basenetworks.py:461-499: squeezenet1_1's features, padded as squeezenet_padding describes."""

    def __init__(self, name='squeezenet'):
        super().__init__()
        import torchvision
        self.name, self.stride, self.out_features = name, 16, 512
        self.backbone = squeezenet_padding(torchvision.models.squeezenet1_1(weights=None)).features

    def forward(self, x):
        return self.backbone(x)


def make_base(name):
    return SqueezeNet(name) if name == 'squeezenet' else ShuffleNetV2(name)


def make_pose_shell(name, seed=0, base=None):
    """the named base + the CocoKp heads (Cif 17, Caf 19 with the COCO person skeleton), seeded as det_models.seed_shell
    seeds (random BatchNorm statistics, eval mode).  SqueezeNet has no BatchNorm: its convs get the He variance 2 /
    fan_in instead of 1 / fan_in, so that 17 ReLU layers keep the activation scale and the features depend on the
    input rather than on the biases alone."""
    base = make_base(name) if base is None else base
    cif, caf = net_oracle.HeadMeta.cif(17), net_oracle.HeadMeta.caf(19)
    caf.skeleton = constants.COCO_PERSON_SKELETON
    heads = [net_oracle.CompositeField4(cif, base.out_features), net_oracle.CompositeField4(caf, base.out_features)]
    shell = det_models.seed_shell(net_oracle.Shell(base, heads), seed)
    if isinstance(base, SqueezeNet):
        with torch.no_grad():
            for m in base.modules():
                if isinstance(m, torch.nn.Conv2d):
                    m.weight.mul_(2.0 ** 0.5)
    return shell


def reference_base(name):
    """The reference's own basenetworks.ShuffleNetV2 / SqueezeNet (pretrained off, torchvision weights=None).  Needs
    the reference sources."""
    import torchvision
    from oracle import make_golden
    _, base, _ = make_golden.load_reference_modules()
    cls = base.SqueezeNet if name == 'squeezenet' else base.ShuffleNetV2
    saved = cls.pretrained
    try:
        cls.pretrained = False
        if name == 'squeezenet':
            return cls(name, lambda pretrained: torchvision.models.squeezenet1_1(weights=None))
        ctor, out_features = SHUFFLENETV2[name]
        return cls(name, lambda pretrained: getattr(torchvision.models, ctor)(weights=None), out_features)
    finally:
        cls.pretrained = saved


def reference_features(name, x, oracle_base):
    """reference_base(name) loaded with the weights of `oracle_base`, applied to x"""
    ref = reference_base(name)
    assert ref.stride == oracle_base.stride == 16 and ref.out_features == oracle_base.out_features
    ref.load_state_dict(oracle_base.state_dict())
    net_oracle.model_defaults(ref)
    ref.eval()
    with torch.no_grad():
        return ref(x)


def golden_inputs():
    """an odd and an even size: at the even one the ceil-mode pools of SqueezeNet add a row and a column"""
    g = torch.Generator().manual_seed(23)
    return {'odd': torch.randn(1, 3, 49, 65, generator=g), 'even': torch.randn(1, 3, 48, 64, generator=g)}

