"""Test infrastructure: fp32 PyTorch restatement of the reference's ShuffleNetV2K with the structural options of its
constructor and CLI, next to oracle/net_oracle.py (paths relative to the reference's src/openpifpaf/):

  ShuffleNetV2K / InvertedResidualK    network/basenetworks.py:186-355
    --shufflenetv2k-stage4-dilation D          stage 4 and conv5-as-stage at stride 1 with dilated depthwise convs
    --shufflenetv2k-input-conv2-stride 2       a second 3x3 stride-2 conv + BN + ReLU in input_block
    --shufflenetv2k-input-conv2-outchannels C  its width (default: the stem's)
    --shufflenetv2k-conv5-as-stage             conv5 = two InvertedResidualK blocks instead of a 1x1 conv

Module attribute names and state_dict keys equal the reference's, so its own modules load these weights unchanged
(tests/test_shufflenetv2k_variants.py compares the two)."""
import torch

import det_models
from openpifpaf_b200 import constants
from oracle import net_oracle

# options of the variants the tests cover (keyword arguments of ShuffleNetV2K)
VARIANTS = {
    'dil2': dict(stage4_dilation=2),
    'conv2': dict(input_conv2_stride=2),
    'conv2_out48': dict(input_conv2_stride=2, input_conv2_outchannels=48),
    'conv5stage': dict(conv5_as_stage=True),
    'dil2_conv5stage': dict(stage4_dilation=2, conv5_as_stage=True),
    'conv2_dil2': dict(input_conv2_stride=2, stage4_dilation=2),
}

# small widths for the CPU tests and the stored features; 'tiny_wide' has a conv5 wider than stage 4, so that
# conv5-as-stage starts with a branch1 block
CONFIGS = {
    'tiny': ([2, 3, 2], [24, 32, 48, 64, 64]),
    'tiny_wide': ([2, 3, 2], [24, 32, 48, 64, 96]),
}
CONFIGS.update(net_oracle.SHUFFLENETV2K_CONFIGS)


class InvertedResidualK(torch.nn.Module):
    """basenetworks.py:186-242 with its stride and dilation options (BatchNorm, ReLU)"""

    def __init__(self, inp, oup, first_in_stage, *, stride=1, dilation=1, kernel_size=5):
        super().__init__()
        assert (stride != 1 or dilation != 1 or inp != oup) or not first_in_stage
        self.first_in_stage = first_in_stage
        bf = oup // 2
        pad = (kernel_size - 1) // 2 * dilation
        bn, relu, conv = torch.nn.BatchNorm2d, (lambda: torch.nn.ReLU(inplace=True)), torch.nn.Conv2d
        self.branch1 = None
        if first_in_stage:
            self.branch1 = torch.nn.Sequential(
                conv(inp, inp, kernel_size, stride, pad, bias=False, groups=inp, dilation=dilation), bn(inp),
                conv(inp, bf, 1, 1, 0, bias=False), bn(bf), relu())
        self.branch2 = torch.nn.Sequential(
            conv(inp if first_in_stage else bf, bf, 1, 1, 0, bias=False), bn(bf), relu(),
            conv(bf, bf, kernel_size, stride, pad, bias=False, groups=bf, dilation=dilation), bn(bf),
            conv(bf, bf, 1, 1, 0, bias=False), bn(bf), relu())

    def forward(self, x):
        if self.branch1 is None:
            x1, x2 = x.chunk(2, dim=1)
            out = torch.cat((x1, self.branch2(x2)), dim=1)
        else:
            out = torch.cat((self.branch1(x), self.branch2(x)), dim=1)
        return net_oracle.channel_shuffle(out, 2)


class ShuffleNetV2K(torch.nn.Module):
    """basenetworks.py:245-355 with the class options of its configure() as keyword arguments; the defaults build
    net_oracle.ShuffleNetV2K."""

    def __init__(self, name, stages_repeats, stages_out_channels, *, stage4_dilation=1, input_conv2_stride=0,
                 input_conv2_outchannels=None, conv5_as_stage=False):
        super().__init__()
        self.name = name
        stride = 16
        c0 = stages_out_channels[0]
        modules = [torch.nn.Sequential(torch.nn.Conv2d(3, c0, 3, 2, 1, bias=False), torch.nn.BatchNorm2d(c0),
                                       torch.nn.ReLU(inplace=True))]
        cin = c0
        if input_conv2_stride:
            c2 = input_conv2_outchannels or cin
            modules.append(torch.nn.Sequential(torch.nn.Conv2d(cin, c2, 3, 2, 1, bias=False), torch.nn.BatchNorm2d(c2),
                                               torch.nn.ReLU(inplace=True)))
            stride *= 2
            cin = c2
        self.input_block = torch.nn.Sequential(*modules)
        stages = []
        for repeats, cout, dil in zip(stages_repeats, stages_out_channels[1:4], (1, 1, stage4_dilation)):
            stage_stride = 2 if dil == 1 else 1
            stride = int(stride * stage_stride / 2)
            seq = [InvertedResidualK(cin, cout, True, stride=stage_stride, dilation=dil)]
            seq += [InvertedResidualK(cout, cout, False, dilation=dil) for _ in range(repeats - 1)]
            stages.append(torch.nn.Sequential(*seq))
            cin = cout
        self.stage2, self.stage3, self.stage4 = stages
        cl = stages_out_channels[-1]
        if conv5_as_stage:
            self.conv5 = torch.nn.Sequential(
                InvertedResidualK(cin, cl, cin != cl, dilation=stage4_dilation),
                InvertedResidualK(cl, cl, False, dilation=stage4_dilation))
        else:
            self.conv5 = torch.nn.Sequential(torch.nn.Conv2d(cin, cl, 1, 1, 0, bias=False), torch.nn.BatchNorm2d(cl),
                                             torch.nn.ReLU(inplace=True))
        self.stride = stride
        self.out_features = cl

    def forward(self, x):
        x = self.input_block(x)
        x = self.stage2(x)
        x = self.stage3(x)
        x = self.stage4(x)
        return self.conv5(x)


def make_base(variant, config='tiny'):
    repeats, channels = CONFIGS[config]
    return ShuffleNetV2K(config, repeats, channels, **VARIANTS[variant])


def make_pose_shell(variant, config='tiny', seed=0):
    """a ShuffleNetV2K variant + the CocoKp heads (Cif 17, Caf 19 with the COCO person skeleton), seeded as
    det_models.seed_shell seeds (variance 1 / fan_in, random BatchNorm statistics, eval mode)"""
    base = make_base(variant, config)
    cif, caf = net_oracle.HeadMeta.cif(17), net_oracle.HeadMeta.caf(19)
    caf.skeleton = constants.COCO_PERSON_SKELETON
    heads = [net_oracle.CompositeField4(cif, base.out_features), net_oracle.CompositeField4(caf, base.out_features)]
    return det_models.seed_shell(net_oracle.Shell(base, heads), seed)


def reference_features(variant, x, oracle_base):
    """The reference's own basenetworks.ShuffleNetV2K with its class attributes set as configure() sets them for
    `variant`, loaded with the weights of `oracle_base`, applied to x.  Needs the reference sources."""
    from oracle import make_golden
    _, base, _ = make_golden.load_reference_modules()
    opts = dict(input_conv2_stride=0, input_conv2_outchannels=None, stage4_dilation=1, conv5_as_stage=False)
    opts.update(VARIANTS[variant])
    saved = {k: getattr(base.ShuffleNetV2K, k) for k in opts}
    try:
        for k, v in opts.items():
            setattr(base.ShuffleNetV2K, k, v)
        repeats, channels = CONFIGS[oracle_base.name]
        ref = base.ShuffleNetV2K(oracle_base.name, repeats, channels)
    finally:
        for k, v in saved.items():
            setattr(base.ShuffleNetV2K, k, v)
    assert ref.stride == oracle_base.stride, (ref.stride, oracle_base.stride)
    ref.load_state_dict(oracle_base.state_dict())
    net_oracle.model_defaults(ref)          # BatchNorm eps as the reference's factory sets it (nets.py:63-78)
    ref.eval()
    with torch.no_grad():
        return ref(x)


def golden_input():
    return torch.randn(1, 3, 49, 65, generator=torch.Generator().manual_seed(23))
