"""Test infrastructure: fp32 PyTorch restatement of the reference's detection models, next to oracle/net_oracle.py
(paths relative to the reference's src/openpifpaf/):

  Resnet with every constructor / CLI option       network/basenetworks.py:71-150
  CompositeField4 with upsample_stride (eval)       network/heads.py:272-378
  headmeta.CifDet                                   headmeta.py:117-125

Module attribute names and state_dict keys equal the reference's, so the reference's modules load these weights
unchanged (tests/test_resnet_variants.py compares the two).  Torchvision is always asked for weights=None: nothing
here downloads a checkpoint."""
import math

import torch

from oracle import net_oracle

# (pool0_stride, input_conv_stride, input_conv2_stride, block5_dilation) of the Resnet variants the tests cover;
# 'cocodet' is the reference guide's resnet18-cocodet recipe (--resnet-input-conv2-stride=2
# --resnet-block5-dilation=2, with the --cocodet-upsample=2 head)
VARIANTS = {
    'default': dict(),
    'pool2': dict(pool0_stride=2),
    'pool1': dict(pool0_stride=1),
    'stem_s1': dict(input_conv_stride=1),
    'conv2': dict(input_conv2_stride=2),
    'dil2': dict(block5_dilation=2),
    'dil4': dict(block5_dilation=4),
    'cocodet': dict(input_conv2_stride=2, block5_dilation=2),
}


class Resnet(torch.nn.Module):
    """basenetworks.py:71-150 with all its class options as constructor arguments."""

    def __init__(self, name, torchvision_resnet, out_features=2048, *, pool0_stride=0, input_conv_stride=2,
                 input_conv2_stride=0, block5_dilation=1, remove_last_block=False):
        super().__init__()
        modules = list(torchvision_resnet(weights=None).children())
        stride = 32
        input_modules = modules[:4]
        if pool0_stride:
            if pool0_stride != 2:
                input_modules[3].stride = torch.nn.modules.utils._pair(pool0_stride)
                stride = int(stride * 2 / pool0_stride)
        else:
            input_modules.pop(3)
            stride //= 2
        if input_conv_stride != 2:
            input_modules[0].stride = torch.nn.modules.utils._pair(input_conv_stride)
            stride = int(stride * 2 / input_conv_stride)
        if input_conv2_stride:
            assert not pool0_stride
            channels = input_modules[0].out_channels
            input_modules.append(torch.nn.Sequential(
                torch.nn.Conv2d(channels, channels, 3, 2, 1, bias=False),
                torch.nn.BatchNorm2d(channels),
                torch.nn.ReLU(inplace=True)))
            stride *= 2
        block5 = modules[7]
        if remove_last_block:
            block5 = None
            stride //= 2
            out_features //= 2
        if block5_dilation != 1:
            stride //= 2
            for m in block5.modules():
                if not isinstance(m, torch.nn.Conv2d):
                    continue
                m.stride = torch.nn.modules.utils._pair(1)
                if m.kernel_size[0] == 1:
                    continue
                m.dilation = torch.nn.modules.utils._pair(block5_dilation)
                m.padding = torch.nn.modules.utils._pair((m.kernel_size[0] - 1) // 2 * block5_dilation)
        self.name = name
        self.stride = stride
        self.out_features = out_features
        self.input_block = torch.nn.Sequential(*input_modules)
        self.block2, self.block3, self.block4, self.block5 = modules[4], modules[5], modules[6], block5

    def forward(self, x):
        x = self.input_block(x)
        x = self.block2(x)
        x = self.block3(x)
        x = self.block4(x)
        return self.block5(x)


def make_resnet(base_name='resnet18', **variant):
    import torchvision
    tv, out = {'resnet18': (torchvision.models.resnet18, 512), 'resnet50': (torchvision.models.resnet50, 2048)}[base_name]
    return Resnet(base_name, tv, out, **variant)


def cifdet_meta(n_categories, upsample_stride=1):
    """headmeta.CifDet (headmeta.py:117-125): one confidence, two vectors (centre with offset, width/height without),
    no scale."""
    m = net_oracle.HeadMeta('cifdet', n_categories, 1, 2, 0, [True, False])
    m.upsample_stride = upsample_stride
    return m


class CompositeField4(net_oracle.CompositeField4):
    """heads.py:272-378 in eval mode including upsample_stride: the conv has n_fields * n_comp * up^2 channels,
    PixelShuffle(up) follows, then the crop of (up - 1) // 2 low and ceil((up - 1) / 2) high cells."""

    def __init__(self, meta, in_features):
        super().__init__(meta, in_features)
        up = meta.upsample_stride
        self.conv = torch.nn.Conv2d(in_features, meta.n_fields * self.n_components * up * up, 1)
        self.upsample_op = torch.nn.PixelShuffle(up) if up > 1 else None

    def forward(self, x):
        m = self.meta
        x = self.conv(x)
        if self.upsample_op is not None:
            x = self.upsample_op(x)
            lo, hi = (m.upsample_stride - 1) // 2, math.ceil((m.upsample_stride - 1) / 2.0)
            x = x[:, :, lo:int(x.shape[2]) - hi, lo:int(x.shape[3]) - hi]
        b, _, h, w = x.shape
        x = x.reshape(b, m.n_fields, self.n_components, h, w)
        torch.sigmoid_(x[:, :, 1:1 + m.n_confidences])
        first_reg = 1 + m.n_confidences
        for i, do_offset in enumerate(m.vector_offsets):
            if do_offset:
                x[:, :, first_reg + i * 2] += torch.arange(w, dtype=x.dtype, device=x.device)
                x[:, :, first_reg + i * 2 + 1] += torch.arange(h, dtype=x.dtype, device=x.device).unsqueeze(1)
        first_scale = 1 + m.n_confidences + m.n_vectors * 2
        scales = x[:, :, first_scale:first_scale + m.n_scales]
        scales[:] = torch.nn.functional.softplus(scales)
        return x


def seed_shell(shell, seed):
    """Reproducible random weights and BatchNorm statistics (eval mode).  Every conv gets variance 1 / fan_in: through
    the ReLUs each residual branch then adds about a quarter of the variance it receives, so the activations grow
    slowly over the blocks and stay input dependent (the He variance 2 / fan_in doubles them at every block)."""
    g = torch.Generator().manual_seed(seed)
    net_oracle.model_defaults(shell)
    with torch.no_grad():
        for m in shell.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) * 0.5 + 0.75)
                m.weight.copy_(torch.rand(m.num_features, generator=g) * 0.5 + 0.75)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)
            elif isinstance(m, torch.nn.Conv2d):
                fan_in = m.weight.shape[1] * m.weight.shape[2] * m.weight.shape[3]
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (1.0 / fan_in) ** 0.5)
                if m.bias is not None:
                    m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
    shell.eval()
    return shell


def make_det_shell(base, n_categories=91, upsample_stride=1, seed=0):
    """A Shell with one CifDet head (as plugins/coco/cocodet.py builds it) on `base`, seeded."""
    head = CompositeField4(cifdet_meta(n_categories, upsample_stride), base.out_features)
    return seed_shell(net_oracle.Shell(base, [head]), seed)


def make_variant_shell(variant, base_name='resnet18', n_keypoints=17, seed=0):
    """A pose Shell (Cif + Caf heads) on the named Resnet variant, seeded; the cocodet variant gets the 91-category
    upsample-2 CifDet head instead."""
    base = make_resnet(base_name, **VARIANTS[variant])
    if variant == 'cocodet':
        return make_det_shell(base, 91, 2, seed)
    heads = [net_oracle.CompositeField4(net_oracle.HeadMeta.cif(n_keypoints), base.out_features),
             net_oracle.CompositeField4(net_oracle.HeadMeta.caf(19), base.out_features)]
    return seed_shell(net_oracle.Shell(base, heads), seed)


def reference_resnet_features(variant, x, oracle_base):
    """The reference's own basenetworks.Resnet, configured like `variant` through its class attributes (as its
    configure() does) and loaded with the weights of `oracle_base`, applied to x.  Needs the reference sources."""
    import torchvision
    from oracle import make_golden
    _, base, _ = make_golden.load_reference_modules()
    opts = dict(pool0_stride=0, input_conv_stride=2, input_conv2_stride=0, block5_dilation=1)
    opts.update(VARIANTS[variant])
    saved = {k: getattr(base.Resnet, k) for k in list(opts) + ['pretrained']}
    try:
        base.Resnet.pretrained = False
        for k, v in opts.items():
            setattr(base.Resnet, k, v)
        assert base.Resnet.pretrained is False
        ref = base.Resnet(oracle_base.name, lambda pretrained: getattr(torchvision.models, oracle_base.name)(weights=None),
                          oracle_base.out_features)
    finally:
        for k, v in saved.items():
            setattr(base.Resnet, k, v)
    assert ref.stride == oracle_base.stride, (ref.stride, oracle_base.stride)
    ref.load_state_dict(oracle_base.state_dict())
    net_oracle.model_defaults(ref)          # BatchNorm eps as the reference's factory sets it (nets.py:63-78)
    ref.eval()
    with torch.no_grad():
        return ref(x)


def golden_variant_input():
    return torch.randn(1, 3, 49, 65, generator=torch.Generator().manual_seed(21))


CONFIDENCE_BIAS, BOX_CELLS = -1.75, 20.0


def calibrate_det_head(shell, confidence_bias=CONFIDENCE_BIAS, box_cells=BOX_CELLS, size=161):
    """Give a from-scratch CifDet head trained-network-like statistics, as network.calibrate_random_heads does for
    plans: centre and rescale every head channel on the features of a probe batch (mean 0, standard deviation 1 over
    positions), add confidence_bias to the confidence channels, shrink the regressions to a tenth and centre the box
    width / height at box_cells cells.  Each image then has detections -- confidence blobs whose votes overlap in the
    CifDetHr map -- instead of a saturated map or scattered votes that never reach the seed threshold."""
    head = shell.head_nets[0]
    up2 = head.meta.upsample_stride ** 2
    dev = next(shell.parameters()).device
    with torch.no_grad():
        feat = shell.base_net(torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(7)).to(dev))
        mu = feat.mean((0, 2, 3))
        w = head.conv.weight[:, :, 0, 0]
        pre = torch.einsum('nc,bchw->bnhw', w, feat - mu[None, :, None, None])
        w = w / pre.std((0, 2, 3))[:, None]
        head.conv.bias.copy_(-(w @ mu))
        head.conv.weight.copy_(w[:, :, None, None])
        wv = head.conv.weight.view(head.meta.n_fields, head.n_components, up2, -1)
        bv = head.conv.bias.view(head.meta.n_fields, head.n_components, up2)
        bv[:, 1] += confidence_bias
        wv[:, 2:6] *= 0.1
        bv[:, 2:6] *= 0.1
        bv[:, 4:6] += box_cells
    return shell
