"""Host-side mirror of the reference network modules for the inference hot path.

Reference (paths relative to the reference's src/openpifpaf/):
  Shell.forward                       network/nets.py:35-48
  ShuffleNetV2K / InvertedResidualK   network/basenetworks.py:186-355
  MobileNetV2 (torchvision features)  network/basenetworks.py:407-417
  ShuffleNetV2 (torchvision x1 / x2)  network/basenetworks.py:36-68
  SqueezeNet (torchvision 1.1)        network/basenetworks.py:461-499
  CompositeField4 (eval)              network/heads.py:330-378

`plan_from_shell(shell)` walks a reference-style ``Shell`` (duck-typed: the
reference's own ``openpifpaf.network.nets.Shell`` or any module tree with the
same attribute names), folds every eval-mode BatchNorm into its convolution and
returns a plain "plan" of float32 numpy arrays.  `CompiledNet` turns a plan into
a fused op list of libpifpaf_b200 (wgmma GEMMs for the 1x1 convolutions) and
replays it.  torch.cat / chunk / channel_shuffle never run as kernels: they are
folded into the physical channel placement computed here.

  'bins' layout (default): every channel of a stage is written once, by the GEMM
  that produces it, into the buffer of the block that consumes it; pass-through
  channels are never copied (see _plan_stage_bins).

  'shuffle' layout: activations in logical channel order; the last GEMM of a block
  writes logical channel 2n <- pass-through[n], 2n+1 <- conv[n] (== cat +
  channel_shuffle(groups=2), basenetworks.py:233-242) with aligned 256-bit stores,
  and the next block's x.chunk(2) is the TMA start coordinate _view_start(half) of
  its A operand (the leading pass-through columns meet zero weight columns).
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib

OP_RAW, OP_SIGMOID, OP_ADD_X, OP_ADD_Y, OP_SOFTPLUS = 0, 1, 2, 3, 4
# activation codes of the conv ops (the `relu` field; include/pifpaf_b200.h)
ACT_NONE, ACT_RELU, ACT_RELU6 = 0, 1, 2

SHUFFLENETV2K_CONFIGS = {     # network/factory.py:68-79
    'shufflenetv2k16': ([4, 8, 4], [24, 348, 696, 1392, 1392]),
    'shufflenetv2k20': ([5, 10, 5], [32, 512, 1024, 2048, 2048]),
    'shufflenetv2k30': ([8, 16, 6], [32, 512, 1024, 2048, 2048]),
}


def pad8(v):
    return (v + 7) // 8 * 8


def pad16(v):
    return (v + 15) // 16 * 16


# ----------------------------------------------------------------------------- plans

class UnsupportedModel(RuntimeError):
    """plan_from_shell refuses the model: a module, option or head the compiled forward does not implement.  Callers
    that have another way to run the model (the plugin's reference fallback) catch this and nothing else."""


def _fold(conv, bn):
    """conv (bias-free) followed by eval BatchNorm -> (weight, bias) float32 numpy.  bn None: the conv alone, its bias
    (zero without one) as the bias (SqueezeNet's convs have biases and no BatchNorm)."""
    w = conv.weight.detach().double()
    if bn is None:
        b = conv.bias.detach().double() if conv.bias is not None else torch.zeros(w.shape[0], dtype=torch.float64)
        return w.float().cpu().numpy(), b.float().cpu().numpy()
    scale = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    b = bn.bias.detach().double() - bn.running_mean.detach().double() * scale
    if conv.bias is not None:
        b = b + conv.bias.detach().double() * scale
    w = w * scale.view(-1, 1, 1, 1)
    return w.float().cpu().numpy(), b.float().cpu().numpy()


def head_ops(n_confidences, n_vectors, n_scales, vector_offsets):
    """Per-component epilogue of CompositeField4.forward in eval mode (heads.py:360-378)."""
    ops = [OP_RAW] + [OP_SIGMOID] * n_confidences
    for i in range(n_vectors):
        ops += [OP_ADD_X, OP_ADD_Y] if vector_offsets[i] else [OP_RAW, OP_RAW]
    ops += [OP_SOFTPLUS] * n_scales
    return ops


def _heads_plan(shell, base):
    heads = []
    for hn in shell.head_nets:
        m = hn.meta
        up = int(getattr(m, 'upsample_stride', 1))
        ncomp = 1 + m.n_confidences + m.n_vectors * 2 + m.n_scales
        heads.append({
            # upsample_stride > 1 (heads.py:307-343): the conv has n_fields * n_comp * up^2 channels, PixelShuffle(up)
            # and the crop run in the GEMM epilogue (pifpaf_net_heads_upsampled)
            'w': hn.conv.weight.detach().float().cpu().numpy().reshape(m.n_fields * ncomp * up * up, -1),
            'b': hn.conv.bias.detach().float().cpu().numpy(),
            'n_fields': int(m.n_fields), 'n_comp': int(ncomp), 'upsample': up,
            'ops': head_ops(m.n_confidences, m.n_vectors, m.n_scales, tuple(m.vector_offsets)),
            'stride': int(base.stride) // up})
    if len({hd['upsample'] for hd in heads}) > 1:
        raise UnsupportedModel('heads with different upsample_stride values are not supported')
    return heads


def _resnet_input_block(input_block):
    """The input block of basenetworks.py:71-150 as [(kind, modules)]: ('conv', (conv, bn)) for each conv + BN + ReLU
    (the stem, and the optional --resnet-input-conv2-stride conv, nested in a Sequential of its own) and ('pool',
    maxpool) for torchvision's max pool kept by --resnet-pool0-stride.  Anything else is refused."""
    mods = []
    for m in input_block:
        mods += list(m) if isinstance(m, torch.nn.Sequential) else [m]
    parts, i = [], 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, torch.nn.Conv2d) and i + 2 < len(mods) and isinstance(mods[i + 1], torch.nn.BatchNorm2d) \
                and isinstance(mods[i + 2], torch.nn.ReLU):
            parts.append(('conv', (m, mods[i + 1])))
            i += 3
        elif isinstance(m, torch.nn.MaxPool2d):
            if (_pair(m.kernel_size), _pair(m.padding), _pair(m.dilation), m.ceil_mode) != ((3, 3), (1, 1), (1, 1), False) \
                    or _pair(m.stride) not in ((1, 1), (2, 2)):
                raise UnsupportedModel('only a 3x3 max pool with padding 1 and stride 1 or 2 is supported')
            parts.append(('pool', m))
            i += 1
        else:
            raise UnsupportedModel(f'unsupported Resnet input block module {type(m).__name__}')
    kinds = [k for k, _ in parts]
    if kinds not in (['conv'], ['conv', 'pool'], ['conv', 'conv']):
        raise UnsupportedModel(f'unsupported Resnet input block {kinds}: expected the stem conv, then a max pool or '
                               'a second conv')
    return parts


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _fold_stem(conv, bn):
    """the stem conv + BN of a ShuffleNetV2K or Resnet input block, folded (its kernel size is the weight's)"""
    w, b = _fold(conv, bn)
    return {'w': w, 'b': b, 'stride': int(conv.stride[0]), 'pad': int(conv.padding[0])}


def _conv_entry(c, n):
    """a square conv + BN, folded, as an implicit-GEMM conv entry; 'dilation' only where it is not 1"""
    if len(set(_pair(c.kernel_size))) != 1 or len(set(_pair(c.stride))) != 1 or \
            len(set(_pair(c.padding))) != 1 or len(set(_pair(c.dilation))) != 1:
        raise UnsupportedModel('only square ResNet convolutions are supported')
    w, b = _fold(c, n)
    e = {'w': w, 'b': b, 'kernel': int(c.kernel_size[0]), 'stride': int(c.stride[0]), 'pad': int(c.padding[0])}
    if c.dilation[0] != 1:
        if c.stride[0] != 1:
            raise UnsupportedModel('dilated convolutions with a stride are not supported')
        e['dilation'] = int(c.dilation[0])
    return e


def _plan_from_resnet(shell):
    """basenetworks.py:71-150: torchvision ResNet (input_block = conv1, bn1, relu, then the max pool under
    --resnet-pool0-stride or a 3x3 conv + BN + ReLU under --resnet-input-conv2-stride; block2..block5 = layer1..layer4
    of BasicBlock / Bottleneck, layer4 dilated under --resnet-block5-dilation)."""
    base = shell.base_net
    if base.block5 is None:
        # basenetworks.py:116-119,149: --resnet-remove-last-block leaves block5 = None, which the reference's own
        # forward then calls
        raise UnsupportedModel('Resnet with remove_last_block (block5 = None) is not supported: its forward fails')
    for m in base.modules():
        if isinstance(m, torch.nn.Conv2d) and m.groups != 1:
            raise UnsupportedModel('grouped convolutions (ResNeXt) are not supported')
    parts = _resnet_input_block(base.input_block)
    plan = {'kind': 'resnet', 'input': _fold_stem(*parts[0][1]), 'blocks': [], 'heads': _heads_plan(shell, base)}
    if len(parts) == 2 and parts[1][0] == 'pool':
        plan['pool'] = {'stride': int(_pair(parts[1][1].stride)[0])}
    elif len(parts) == 2:
        plan['input2'] = _conv_entry(*parts[1][1])

    for stage in (base.block2, base.block3, base.block4, base.block5):
        for blk in stage:
            e = {'convs': [_conv_entry(blk.conv1, blk.bn1), _conv_entry(blk.conv2, blk.bn2)]}
            if hasattr(blk, 'conv3'):
                e['convs'].append(_conv_entry(blk.conv3, blk.bn3))
            e['downsample'] = None if blk.downsample is None else _conv_entry(blk.downsample[0], blk.downsample[1])
            plan['blocks'].append(e)
    return plan


def _conv_bn_relu6(m, what):
    """torchvision's Conv2dNormActivation (ConvBNReLU in older releases) with ReLU6 -> (conv, bn)"""
    parts = list(m) if isinstance(m, torch.nn.Sequential) else []
    if len(parts) != 3 or not isinstance(parts[0], torch.nn.Conv2d) or not isinstance(parts[1], torch.nn.BatchNorm2d):
        raise UnsupportedModel(f'MobileNetV2 {what}: expected Conv2d + BatchNorm2d + ReLU6, got {type(m).__name__}')
    if not isinstance(parts[2], torch.nn.ReLU6):
        raise UnsupportedModel(f'MobileNetV2 {what}: unsupported activation {type(parts[2]).__name__} (only ReLU6)')
    return parts[0], parts[1]


def _mobilenet_conv(conv, bn, what, kernel, stride=None, depthwise=False):
    """one conv of the MobileNetV2 backbone, checked against the shapes torchvision builds, folded"""
    k, s, p, d = _pair(conv.kernel_size), _pair(conv.stride), _pair(conv.padding), _pair(conv.dilation)
    groups_ok = conv.groups == conv.in_channels == conv.out_channels if depthwise else conv.groups == 1
    if k != (kernel, kernel) or s[0] != s[1] or s[0] not in ((1, 2) if stride is None else (stride,)) or \
            p != ((kernel - 1) // 2,) * 2 or d != (1, 1) or not groups_ok:
        raise UnsupportedModel(f'MobileNetV2 {what}: unsupported conv {conv}')
    # torchvision rounds every width to a multiple of 8 (_make_divisible); the channel padding of the lowering
    # (16-channel rows, 8-channel depthwise vectors) is laid out for that
    if conv.out_channels % 8 or (conv.in_channels % 8 and conv.in_channels != 3):
        raise UnsupportedModel(f'MobileNetV2 {what}: channel counts must be multiples of 8, got {conv}')
    w, b = _fold(conv, bn)
    return {'w': w, 'b': b, 'kernel': kernel, 'stride': int(s[0]), 'pad': (kernel - 1) // 2}


def _plan_from_mobilenetv2(shell):
    """basenetworks.py:407-417: base_net.backbone = torchvision mobilenet_v2().features -- the 3x3 stride-2 stem,
    17 InvertedResidual blocks (1x1 expand + ReLU6 unless the expansion is 1, 3x3 depthwise + ReLU6, 1x1 linear
    projection, plus the block input when stride 1 and in == out) and the final 1x1 conv + ReLU6; stride 32."""
    base = shell.base_net
    mods = list(base.backbone)
    if len(mods) < 3:
        raise UnsupportedModel('MobileNetV2 backbone: expected a stem, InvertedResidual blocks and a last conv')
    conv, bn = _conv_bn_relu6(mods[0], 'stem')
    stem = _mobilenet_conv(conv, bn, 'stem', 3, 2)
    if conv.in_channels != 3:
        raise UnsupportedModel('MobileNetV2 stem: expected 3 input channels')
    blocks = []
    for i, m in enumerate(mods[1:-1], start=1):
        layers = list(m.conv) if isinstance(getattr(m, 'conv', None), torch.nn.Sequential) else []
        if not hasattr(m, 'use_res_connect') or len(layers) not in (3, 4) or \
                not isinstance(layers[-2], torch.nn.Conv2d) or not isinstance(layers[-1], torch.nn.BatchNorm2d):
            raise UnsupportedModel(f'MobileNetV2 backbone[{i}]: expected an InvertedResidual, got {type(m).__name__}')
        what = f'backbone[{i}]'
        e = {'expand': _mobilenet_conv(*_conv_bn_relu6(layers[0], what), what, 1) if len(layers) == 4 else None}
        e['dw'] = _mobilenet_conv(*_conv_bn_relu6(layers[-3], what), what, 3, depthwise=True)
        e['project'] = _mobilenet_conv(layers[-2], layers[-1], what, 1, 1)
        c_in = e['expand']['w'].shape[1] if e['expand'] is not None else e['dw']['w'].shape[0]
        e['residual'] = bool(m.use_res_connect)
        if e['residual'] != (e['dw']['stride'] == 1 and c_in == e['project']['w'].shape[0]):
            raise UnsupportedModel(f'MobileNetV2 {what}: residual connection does not match stride and widths')
        blocks.append(e)
    conv, bn = _conv_bn_relu6(mods[-1], 'last conv')
    last = _mobilenet_conv(conv, bn, 'last conv', 1, 1)
    return {'kind': 'mobilenetv2', 'input': stem, 'blocks': blocks, 'last': last, 'heads': _heads_plan(shell, base)}


def _conv_bn_relu(m, what, kernel, stride, pad):
    """a Sequential of Conv2d (kernel, stride, pad, groups 1) + BatchNorm2d + ReLU -> (conv, bn)"""
    parts = list(m) if isinstance(m, torch.nn.Sequential) else []
    if len(parts) != 3 or not isinstance(parts[0], torch.nn.Conv2d) or not isinstance(parts[1], torch.nn.BatchNorm2d) \
            or not isinstance(parts[2], torch.nn.ReLU):
        raise UnsupportedModel(f'ShuffleNetV2 {what}: expected Conv2d + BatchNorm2d + ReLU')
    c = parts[0]
    if (_pair(c.kernel_size), _pair(c.stride), _pair(c.padding), _pair(c.dilation), c.groups) != \
            ((kernel, kernel), (stride, stride), (pad, pad), (1, 1), 1):
        raise UnsupportedModel(f'ShuffleNetV2 {what}: unsupported conv {c}')
    return parts[0], parts[1]


def _plan_from_shufflenetv2(shell):
    """basenetworks.py:36-68: torchvision's ShuffleNetV2 (x1 / x2) without its max pool -- conv1 (3x3 stride-2 conv +
    BN + ReLU), stages 2-4 of torchvision InvertedResidual blocks (InvertedResidualK with 3x3 depthwise convs and the
    same Sequential indices; a stride-1 block has an empty branch1) and conv5 (1x1 conv + BN + ReLU); stride 16.  The
    plan is a ShuffleNetV2K plan, so it takes that lowering."""
    base = shell.base_net
    conv, bn = _conv_bn_relu(base.conv1, 'conv1', 3, 2, 1)
    if conv.in_channels != 3:
        raise UnsupportedModel('ShuffleNetV2 conv1: expected 3 input channels')
    plan = {'kind': 'shufflenetv2k', 'input': _fold_stem(conv, bn), 'stages': [], 'heads': []}
    for stage in (base.stage2, base.stage3, base.stage4):
        plan['stages'].append([_shufflenetv2k_block(blk) for blk in stage])
    plan['conv5'] = _fold(*_conv_bn_relu(base.conv5, 'conv5', 1, 1, 0))
    plan['heads'] = _heads_plan(shell, base)
    return plan


def _is_fire(m):
    return all(hasattr(m, a) for a in ('squeeze', 'expand1x1', 'expand3x3'))


def _squeezenet_conv(conv, act, what, kernel):
    """one conv of a Fire module (or the stem) with its activation: stride 1 (the stem: 2), padding (kernel - 1) // 2 as
    the reference sets it, groups 1, a ReLU, and a width the column windows of the lowering can hold"""
    stride = 2 if what == 'stem' else 1
    if not isinstance(conv, torch.nn.Conv2d) or (_pair(conv.kernel_size), _pair(conv.stride), _pair(conv.padding),
                                                 _pair(conv.dilation)) != \
            ((kernel, kernel), (stride, stride), ((kernel - 1) // 2,) * 2, (1, 1)):
        raise UnsupportedModel(f'SqueezeNet {what}: unsupported conv {conv}')
    if conv.groups != 1:
        raise UnsupportedModel(f'SqueezeNet {what}: grouped convolutions are not supported')
    if not isinstance(act, torch.nn.ReLU):
        raise UnsupportedModel(f'SqueezeNet {what}: expected a ReLU, got {type(act).__name__}')
    # the expand pair writes one tensor through two column windows that start at multiples of 8 channels
    if conv.out_channels % 8 or (conv.in_channels % 8 and what != 'stem'):
        raise UnsupportedModel(f'SqueezeNet {what}: widths must be multiples of 8, got {conv}')
    w, b = _fold(conv, None)
    return {'w': w, 'b': b, 'kernel': kernel, 'stride': stride, 'pad': (kernel - 1) // 2}


def _plan_from_squeezenet(shell):
    """basenetworks.py:461-499: base_net.backbone = torchvision squeezenet1_1().features with the reference's padding
    edits -- the 3x3 stride-2 stem (pad 1) + ReLU, three 3x3 stride-2 max pools (pad 1, ceil_mode) and eight Fire
    modules (squeeze 1x1 + ReLU, then cat(expand1x1 + ReLU, expand3x3 (pad 1) + ReLU)); convs with biases, no
    BatchNorm; stride 16.  plan['layers'] holds {'type': 'pool', 'stride', 'ceil_mode'} and {'type': 'fire',
    'squeeze', 'expand1x1', 'expand3x3'} in order."""
    base = shell.base_net
    mods = list(base.backbone)
    if len(mods) < 3 or not isinstance(mods[0], torch.nn.Conv2d):
        raise UnsupportedModel('SqueezeNet backbone: expected a stem conv + ReLU, then max pools and Fire modules')
    stem = _squeezenet_conv(mods[0], mods[1], 'stem', 3)
    if mods[0].in_channels != 3:
        raise UnsupportedModel('SqueezeNet stem: expected 3 input channels')
    layers = []
    for i, m in enumerate(mods[2:], start=2):
        what = f'backbone[{i}]'
        if isinstance(m, torch.nn.MaxPool2d):
            if (_pair(m.kernel_size), _pair(m.padding), _pair(m.dilation)) != ((3, 3), (1, 1), (1, 1)) or \
                    _pair(m.stride) not in ((1, 1), (2, 2)):
                raise UnsupportedModel(f'SqueezeNet {what}: only a 3x3 max pool with padding 1 and stride 1 or 2 is '
                                       'supported')
            layers.append({'type': 'pool', 'stride': int(_pair(m.stride)[0]), 'ceil_mode': bool(m.ceil_mode)})
        elif _is_fire(m):
            acts = [getattr(m, a, None) for a in ('squeeze_activation', 'expand1x1_activation', 'expand3x3_activation')]
            layers.append({'type': 'fire', 'squeeze': _squeezenet_conv(m.squeeze, acts[0], f'{what}.squeeze', 1),
                           'expand1x1': _squeezenet_conv(m.expand1x1, acts[1], f'{what}.expand1x1', 1),
                           'expand3x3': _squeezenet_conv(m.expand3x3, acts[2], f'{what}.expand3x3', 3)})
            # the expand3x3 half is written from column e1: pifpaf_net_conv starts an output window on a 16-channel
            # (32-byte) boundary
            if m.expand1x1.out_channels % 16:
                raise UnsupportedModel(f'SqueezeNet {what}.expand1x1: the expand3x3 half would start at column '
                                       f'{m.expand1x1.out_channels}, not a multiple of 16')
        else:
            raise UnsupportedModel(f'SqueezeNet {what}: expected a MaxPool2d or a Fire module, got {type(m).__name__}')
    return {'kind': 'squeezenet', 'input': stem, 'layers': layers, 'heads': _heads_plan(shell, base)}


def plan_from_shell(shell):
    """Extract a folded plan from a reference-style Shell (ShuffleNetV2K, Resnet, MobileNetV2, torchvision ShuffleNetV2
    or SqueezeNet base net)."""
    base = shell.base_net
    if shell.training:
        raise UnsupportedModel('the Shell must be in eval() mode (BatchNorm is folded)')
    # network/nets.py:12-13,36-46: optional pre/post-processing hooks -- not lowered, so refuse them loudly
    if getattr(shell, 'process_input', None) is not None or getattr(shell, 'process_heads', None) is not None:
        raise UnsupportedModel('Shell.process_input / process_heads are not supported by the compiled forward')
    for m in base.modules():
        # the kernels fuse max(x, 0); --shufflenetv2k-leaky-relu etc. would be folded wrongly
        if isinstance(m, (torch.nn.LeakyReLU, torch.nn.ELU, torch.nn.PReLU, torch.nn.SiLU, torch.nn.GELU,
                          torch.nn.Hardswish, torch.nn.InstanceNorm2d, torch.nn.GroupNorm)):
            raise UnsupportedModel(f'unsupported module in the base network: {type(m).__name__} (only ReLU + BatchNorm)')
    if all(hasattr(base, a) for a in ('input_block', 'block2', 'block3', 'block4', 'block5')):
        return _plan_from_resnet(shell)
    # SqueezeNet keeps its layers in base.backbone as MobileNetV2 does: its Fire modules tell them apart
    if isinstance(getattr(base, 'backbone', None), torch.nn.Sequential) and any(_is_fire(m) for m in base.backbone):
        return _plan_from_squeezenet(shell)
    if isinstance(getattr(base, 'backbone', None), torch.nn.Sequential):
        return _plan_from_mobilenetv2(shell)
    if all(hasattr(base, a) for a in ('conv1', 'stage2', 'stage3', 'stage4', 'conv5')):
        return _plan_from_shufflenetv2(shell)
    if not all(hasattr(base, a) for a in ('input_block', 'stage2', 'stage3', 'stage4', 'conv5')):
        raise UnsupportedModel(f'unsupported base network {type(base).__name__}: expected ShuffleNetV2K, Resnet or '
                               'MobileNetV2')
    return _plan_from_shufflenetv2k(shell)


def _shufflenetv2k_block(blk):
    """one InvertedResidualK (basenetworks.py:186-242) or torchvision InvertedResidual (the same Sequential indices; its
    stride-1 blocks have an empty branch1 where InvertedResidualK has None), folded; 'dilation' only where it is not 1
    (--shufflenetv2k-stage4-dilation, which the reference pairs with stride 1)"""
    b2 = blk.branch2
    dw = b2[3]
    first = blk.branch1 is not None and len(blk.branch1) > 0
    entry = {'first': first, 'stride': int(dw.stride[0]),
             'kernel': int(dw.kernel_size[0]), 'pad': int(dw.padding[0])}
    if dw.dilation[0] != 1:
        if entry['stride'] != 1:
            raise UnsupportedModel('dilated depthwise convolutions with a stride are not supported')
        entry['dilation'] = int(dw.dilation[0])
    entry['b2_pw1'] = _fold(b2[0], b2[1])
    entry['b2_dw'] = _fold(b2[3], b2[4])
    entry['b2_pw2'] = _fold(b2[5], b2[6])
    if first:
        entry['b1_dw'] = _fold(blk.branch1[0], blk.branch1[1])
        entry['b1_pw'] = _fold(blk.branch1[2], blk.branch1[3])
    return entry


def _plan_from_shufflenetv2k(shell):
    """basenetworks.py:245-355: the stem (and the second 3x3 stride-2 conv of --shufflenetv2k-input-conv2-stride as
    plan['input2']), stages 2-4 (stage 4 at stride 1 with dilated depthwise convs under
    --shufflenetv2k-stage4-dilation) and conv5: a 1x1 conv (plan['conv5']) or, under --shufflenetv2k-conv5-as-stage,
    two more InvertedResidualK blocks (plan['conv5_stage'])."""
    base = shell.base_net
    if len(base.input_block) not in (1, 2):
        raise UnsupportedModel(f'unsupported ShuffleNetV2K input block of {len(base.input_block)} convolutions')
    plan = {'kind': 'shufflenetv2k', 'input': _fold_stem(base.input_block[0][0], base.input_block[0][1]),
            'stages': [], 'heads': []}
    if len(base.input_block) == 2:
        conv, bn = base.input_block[1][0], base.input_block[1][1]
        if _pair(conv.kernel_size) != (3, 3) or _pair(conv.stride) != (2, 2) or _pair(conv.padding) != (1, 1) or \
                _pair(conv.dilation) != (1, 1) or conv.groups != 1:
            raise UnsupportedModel(f'ShuffleNetV2K input_conv2: expected a 3x3 stride-2 conv, got {conv}')
        plan['input2'] = _conv_entry(conv, bn)
    for stage in (base.stage2, base.stage3, base.stage4):
        plan['stages'].append([_shufflenetv2k_block(blk) for blk in stage])
    if isinstance(base.conv5[0], torch.nn.Conv2d):
        plan['conv5'] = _fold(base.conv5[0], base.conv5[1])
    else:
        plan['conv5_stage'] = [_shufflenetv2k_block(blk) for blk in base.conv5]
    plan['heads'] = _heads_plan(shell, base)
    return plan


def heads_only_plan(plan, c_in=None):
    """The heads of `plan` as a net of their own (one GEMM with the CompositeField4 eval epilogue); compile it with
    the FEATURE map size as in_h, in_w and run it with CompiledNet.forward_features."""
    c = int(plan['heads'][0]['w'].shape[1]) if c_in is None else int(c_in)
    return {'kind': 'heads_only', 'c_in': c, 'heads': plan['heads']}


def random_plan(base_name='shufflenetv2k16', heads=((17, 1, 1, 1), (19, 1, 2, 2)), seed=0, confidence_bias=-4.0, *,
                stage4_dilation=1, input_conv2_stride=0, input_conv2_outchannels=None, conv5_as_stage=False):
    """Random-init folded plan of the named architecture (no checkpoint can be downloaded here).
    heads: (n_fields, n_confidences, n_vectors, n_scales) per head; vector offsets all True.
    confidence_bias is added to the bias of the confidence channels so that a random-init head emits a
    sparse confidence map (sigmoid(-4) ~ 0.02) like a trained network's background; with a zero bias every
    cell sits near 0.5 and passes every decoder threshold, which no trained model produces.
    The keyword options are the reference's --shufflenetv2k-stage4-dilation, --shufflenetv2k-input-conv2-stride,
    --shufflenetv2k-input-conv2-outchannels and --shufflenetv2k-conv5-as-stage (basenetworks.py:245-334); the plan has
    the layout `plan_from_shell` extracts from such a Shell."""
    repeats, ch = SHUFFLENETV2K_CONFIGS[base_name]
    rng = np.random.Generator(np.random.PCG64(seed))

    def conv(cout, cin, k=1, dw=False):
        fan_in = (1 if dw else cin) * k * k
        w = rng.standard_normal((cout, 1 if dw else cin, k, k)).astype(np.float32) * np.float32(np.sqrt(2.0 / fan_in))
        b = (rng.standard_normal(cout) * 0.05).astype(np.float32)
        return w, b

    def block(cin, cout, first, stride, dil):
        bf = cout // 2
        e = {'first': first, 'stride': stride, 'kernel': 5, 'pad': 2 * dil}
        if dil != 1:
            e['dilation'] = dil
        e['b2_pw1'] = conv(bf, cin if first else bf)
        e['b2_dw'] = conv(bf, bf, 5, dw=True)
        e['b2_pw2'] = conv(bf, bf)
        if first:
            e['b1_dw'] = conv(cin, cin, 5, dw=True)
            e['b1_pw'] = conv(bf, cin)
        return e

    w, b = conv(ch[0], 3, 3)
    plan = {'kind': 'shufflenetv2k', 'input': {'w': w, 'b': b, 'stride': 2, 'pad': 1}, 'stages': [], 'heads': []}
    cin = ch[0]
    stride = 16                     # basenetworks.py:271-313
    if input_conv2_stride:
        c2 = input_conv2_outchannels or cin
        w, b = conv(c2, cin, 3)
        plan['input2'] = {'w': w, 'b': b, 'kernel': 3, 'stride': 2, 'pad': 1}
        cin, stride = c2, stride * 2
    for rep, cout, dil in zip(repeats, ch[1:4], (1, 1, stage4_dilation)):
        if dil != 1:
            stride //= 2
        plan['stages'].append([block(cin if i == 0 else cout, cout, i == 0, 2 if i == 0 and dil == 1 else 1, dil)
                               for i in range(rep)])
        cin = cout
    if conv5_as_stage:
        plan['conv5_stage'] = [block(cin, ch[4], cin != ch[4], 1, stage4_dilation),
                               block(ch[4], ch[4], False, 1, stage4_dilation)]
    else:
        plan['conv5'] = conv(ch[4], cin)
    plan['heads'] = _random_heads(rng, heads, ch[4], stride, confidence_bias)
    return plan


def _random_heads(rng, heads, c_in, stride, confidence_bias, upsample=1):
    """Random-init heads on c_in features at the given feature stride, drawn from rng (weights, then biases, head by
    head).  A head spec is (n_fields, n_confidences, n_vectors, n_scales), optionally with the vector offsets as a
    fifth entry (default: every vector has one).  upsample is the heads' upsample_stride."""
    out = []
    for spec in heads:
        nf, nconf, nvec, nsc = spec[:4]
        offsets = tuple(spec[4]) if len(spec) > 4 else (True,) * nvec
        ncomp = 1 + nconf + 2 * nvec + nsc
        nc = nf * ncomp * upsample * upsample
        w = (rng.standard_normal((nc, c_in)) * np.sqrt(1.0 / c_in)).astype(np.float32)
        b = (rng.standard_normal(nc) * 0.1).astype(np.float32)
        # conv channel (field * n_comp + comp) * up^2 + sub (PixelShuffle order, heads.py:333-343)
        b.reshape(nf, ncomp, upsample * upsample)[:, 1:1 + nconf] += np.float32(confidence_bias)
        hd = {'w': w, 'b': b, 'n_fields': nf, 'n_comp': ncomp,
              'ops': head_ops(nconf, nvec, nsc, offsets), 'stride': stride // upsample}
        if upsample != 1:
            hd['upsample'] = upsample
        out.append(hd)
    return out


RESNET_CONFIGS = {      # torchvision.models.resnet: (block, layers); network/factory.py:57-58
    'resnet18': ('basic', [2, 2, 2, 2]),
    'resnet50': ('bottleneck', [3, 4, 6, 3]),
}


def random_resnet_plan(base_name='resnet50', heads=((17, 1, 1, 1), (19, 1, 2, 2)), seed=0, confidence_bias=-4.0, *,
                       pool0_stride=0, input_conv_stride=2, input_conv2_stride=0, block5_dilation=1, upsample=1):
    """Random-init folded plan of the reference's Resnet base network (basenetworks.py:71-150: torchvision ResNet,
    max-pool removed, stride 16; BasicBlock 3x3-3x3 / Bottleneck 1x1-3x3(stride)-1x1 with expansion 4, 1x1
    downsample on the first block of a stage) -- the same dict layout `_plan_from_resnet` extracts from a Shell.
    The last conv of a block and the downsample conv get half the He variance so that the residual sum keeps the
    activation scale over 16 blocks.  The keyword options are the reference's --resnet-pool0-stride,
    --resnet-input-conv-stride, --resnet-input-conv2-stride and --resnet-block5-dilation; upsample is the heads'
    upsample_stride (--cocodet-upsample).  A head may carry its vector offsets as a fifth entry (CifDet:
    (n_categories, 1, 2, 0, (True, False))); without it every vector has an offset."""
    kind, layers = RESNET_CONFIGS[base_name]
    rng = np.random.Generator(np.random.PCG64(seed))

    def conv(cout, cin, k, stride, gain=2.0, dilation=1):
        w = rng.standard_normal((cout, cin, k, k)).astype(np.float32) * np.float32(np.sqrt(gain / (cin * k * k)))
        b = (rng.standard_normal(cout) * 0.05).astype(np.float32)
        e = {'w': w, 'b': b, 'kernel': k, 'stride': stride, 'pad': (k - 1) // 2 * dilation}
        if dilation != 1:
            e['dilation'] = dilation
        return e

    stem = conv(64, 3, 7, input_conv_stride)
    plan = {'kind': 'resnet', 'input': {'w': stem['w'], 'b': stem['b'], 'stride': input_conv_stride, 'pad': 3},
            'blocks': [], 'heads': []}
    # output stride as basenetworks.py:79-128 tracks it: 32, times 2 / pool stride (16 without the pool), times
    # 2 / input conv stride, times 2 with the second input conv, halved by block5 dilation
    base_stride = 32 * 2 // pool0_stride if pool0_stride else 16
    base_stride = base_stride * 2 // input_conv_stride
    if pool0_stride:
        plan['pool'] = {'stride': pool0_stride}
    if input_conv2_stride:
        plan['input2'] = conv(64, 64, 3, 2)         # Conv2d(channels, channels, 3, 2, 1), basenetworks.py:100-112
        base_stride *= 2
    if block5_dilation != 1:
        base_stride //= 2
    expansion = 1 if kind == 'basic' else 4
    cin = 64
    for si, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
        dil = block5_dilation if si == 3 else 1
        for bi in range(n):
            stride = 2 if (bi == 0 and si > 0 and dil == 1) else 1
            cout = planes * expansion
            if kind == 'basic':
                convs = [conv(planes, cin, 3, stride, dilation=dil), conv(planes, planes, 3, 1, gain=1.0, dilation=dil)]
            else:
                convs = [conv(planes, cin, 1, 1), conv(planes, planes, 3, stride, dilation=dil),
                         conv(cout, planes, 1, 1, gain=1.0)]
            down = conv(cout, cin, 1, stride, gain=1.0) if (stride != 1 or cin != cout) else None
            plan['blocks'].append({'convs': convs, 'downsample': down})
            cin = cout
    plan['heads'] = _random_heads(rng, heads, cin, base_stride, confidence_bias, upsample)
    return plan


def calibrate_random_heads(plan, device=0, seed=0, size=161, batch=2):
    """Give a random-init plan trained-network-like head statistics: measure mean and spread of the backbone
    features on a small random batch (on the GPU, through the product kernels), then centre and rescale the head
    so that every head channel's pre-activation is ~N(0, 1) over positions: w' = w / std, b' = b - w' . mean.
    (Post-ReLU features have a large common mean; without centring every head channel gets its own random DC
    offset and whole confidence maps saturate.)  Together with random_plan's confidence bias this yields
    confidence maps with isolated cells above the decoder thresholds instead of saturated noise.
    Returns (feature std, feature mean norm)."""
    net = CompiledNet(plan, size, size, batch, device=device)
    x = torch.randn((batch, 3, size, size), generator=torch.Generator().manual_seed(seed)).to(f'cuda:{device}')
    net.forward(x)
    torch.cuda.synchronize()
    t, lay = net.info['feature']
    feat = net.tap(t, batch)[..., lay.cols()].astype(np.float64)
    mu = feat.reshape(-1, feat.shape[-1]).mean(axis=0)
    std = float(np.sqrt(np.mean(np.square(feat - mu))))
    for hd in plan['heads']:
        w = hd['w'].astype(np.float64) / max(std, 1e-6)
        hd['b'] = (hd['b'].astype(np.float64) - w @ mu).astype(np.float32)
        hd['w'] = w.astype(np.float32)
    return std, float(np.linalg.norm(mu))


# ----------------------------------------------------------------------------- compiled net

class _DevArray:
    """Expose a raw device pointer to torch through __cuda_array_interface__ (no copy)."""

    def __init__(self, ptr, shape, typestr='<f4'):
        self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': typestr, 'data': (int(ptr), False),
                                         'version': 2}


class _Layout:
    """Physical column placement of a logical channel vector; rows padded to a multiple of 16 channels (32-byte
    aligned rows for 256-bit stores).  Default: physical == logical order.  `split` marks tensors of the
    'shuffle' layout whose two logical halves are consumed separately (x.chunk(2)): the second half starts at
    column `half`; its TMA view starts at _view_start(half) with zero weights on the leading columns.
    `phys` (int array [channels]) places logical channel c at physical column phys[c] of a `width`-wide row (the
    'bins' layout's stage outputs, whose rows hold the channels in order of production)."""

    def __init__(self, channels, split, phys=None, width=None):
        self.channels = channels
        self.split = split
        self.half = channels // 2 if split else None
        self.width = pad16(channels) if width is None else width
        self.phys = None if phys is None else np.asarray(phys, dtype=np.int64)

    def cols(self):
        return np.arange(self.channels) if self.phys is None else self.phys


def _view_start(half):
    """First column of the x.chunk(2)[1] view: a multiple of 8 channels (16 bytes, the TMA requirement), aligned
    further down (to 64 / 32 / 16 channels) as long as the GEMM keeps its number of 64-channel K blocks -- a box
    row that starts on a 128-byte line costs one L2 request instead of two."""
    align = os.environ.get('PIFPAF_VIEW_ALIGN', 'auto')
    if align != 'auto':
        return half // int(align) * int(align)
    k_blocks = (half - half // 8 * 8 + half + 63) // 64
    for al in (64, 32, 16, 8):
        a0 = half // al * al
        if (half - a0 + half + 63) // 64 == k_blocks:
            return a0
    return half // 8 * 8


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _plan_stage_bins(bf, n_blocks):
    """Channel routing of one ShuffleNetV2K stage for the 'bins' layout, in which no pass-through channel is ever
    copied.  The reference (basenetworks.py:233-242) computes, for block t >= 1 with input vector L_t (2*bf
    channels), L_{t+1}[2n] = L_t[n] (pass-through) and L_{t+1}[2n+1] = branch2(L_t[bf:])[n]; block 0 gives
    L_1[2n] = branch1[n], L_1[2n+1] = branch2[n].  So a channel born at position p of L_v sits at position
    p * 2^(t-v) of L_t until that position reaches bf: then it is an input of block t's branch2 (weight column
    position - bf) and dies; channels that never reach bf live on into L_T, the stage output.
    Every channel is therefore WRITTEN ONCE, by its producer GEMM, straight into the buffer of the block that
    consumes it ("bin" t = the bf inputs of block t, or the stage output), and never moved: the producer GEMM's
    columns are ordered by destination, each destination piece padded to a multiple of 16 channels (32 bytes:
    whole sectors, one 256-bit store per lane and 16 columns).

    Producers: 0 = branch1 of block 0, 1 = branch2 of block 0, t + 1 = branch2 of block t (1 <= t < n_blocks).
    Returns (producers, bins, final):
      producers[k] = {'order': int[n_total] (GEMM column -> producer output channel, -1 padding),
                      'pieces': [(col0, count, dest, dest_col)], dest = block index t or 'final'}
      bins[t]      = {'width': W (multiple of 16), 'wcol': int[W] (slot -> weight column of block t's first 1x1, -1 padding)}
      final        = {'width': W, 'logical': int[W] (slot -> channel index of the stage output, -1 padding)}"""
    T = n_blocks
    # piece granularity in channels (16 = 32 bytes: whole sectors).  PIFPAF_BIN_PAD=32 makes every piece a whole number of
    # 64-byte DRAM bursts (more padding columns)
    G = int(os.environ.get('PIFPAF_BIN_PAD', '16'))

    def route(v, p):
        for t in range(max(v, 1), T):
            pos = p << (t - v)
            if pos >= bf:
                return t, pos - bf
        return 'final', p << (T - v)

    births = [(1, [2 * n for n in range(bf)]), (1, [2 * n + 1 for n in range(bf)])]
    births += [(t + 1, [2 * n + 1 for n in range(bf)]) for t in range(1, T)]
    dest_fill = {t: 0 for t in range(1, T)}
    dest_fill['final'] = 0
    slots = {d: [] for d in dest_fill}              # dest -> list of (dest_col, values) pieces
    producers = []
    for v, positions in births:
        routed = [route(v, p) for p in positions]
        order, pieces = [], []
        for d in list(range(1, T)) + ['final']:
            members = [n for n in range(bf) if routed[n][0] == d]
            if not members:
                continue
            padded = (len(members) + G - 1) // G * G
            pieces.append((len(order), padded, d, dest_fill[d]))
            slots[d].append((dest_fill[d], [routed[n][1] for n in members] + [-1] * (padded - len(members))))
            order += members + [-1] * (padded - len(members))
            dest_fill[d] += padded
        producers.append({'order': np.asarray(order, dtype=np.int64), 'pieces': pieces})

    def flat(d):
        out = np.full((dest_fill[d],), -1, dtype=np.int64)
        for col, vals in slots[d]:
            out[col:col + len(vals)] = vals
        return out

    bins = {t: {'width': dest_fill[t], 'wcol': flat(t)} for t in range(1, T)}
    final = {'width': dest_fill['final'], 'logical': flat('final')}
    for t in range(1, T):
        assert sorted(int(c) for c in bins[t]['wcol'] if c >= 0) == list(range(bf))
    assert sorted(int(c) for c in final['logical'] if c >= 0) == list(range(2 * bf))
    return producers, bins, final


def _branch_pitch(bf):
    """Physical channel count of the branch-internal tensors (1x1 -> depthwise -> 1x1).  The depthwise kernels fetch
    one 64-channel block (128 bytes) per pixel and CTA; with a pitch that is a multiple of 64 channels every block is
    one aligned 128-byte line instead of straddling two 64-byte DRAM atoms.  PIFPAF_BRANCH_PAD selects the multiple
    (16: the round-1 layout)."""
    mult = int(os.environ.get('PIFPAF_BRANCH_PAD', '16'))
    return (bf + mult - 1) // mult * mult


def _dw_in_pitch(bf):
    """Physical channel count of the tensor BETWEEN the first 1x1 of a branch and its depthwise conv.  DRAM serves the
    depthwise kernels' TMA reads (one 128-byte 64-channel block per pixel) in aligned 128-byte lines: with 352- / 704-byte
    pixels (176 / 352 channels) a block straddles two lines and the launch reads 1.96x / 1.55x the tensor
    ; tensors whose pixels are a multiple of 128 bytes read 1.00x.  Only this tensor
    is padded (to 64 channels): its producer writes the real channels with the same stores as before, and the tensor
    behind the depthwise conv -- the A operand of a GEMM, which would read the padding -- keeps the 16-channel pitch.
    PIFPAF_DWIN_PAD selects the multiple (16 = the old layout)."""
    mult = int(os.environ.get('PIFPAF_DWIN_PAD', '64'))
    return max(_branch_pitch(bf), (bf + mult - 1) // mult * mult)


def default_layout():
    """'bins' (no pass-through copies, see _plan_stage_bins) or 'shuffle' (every block writes the interleaved
    2*bf-channel tensor through the fused cat+shuffle epilogue); PIFPAF_LAYOUT overrides."""
    return os.environ.get('PIFPAF_LAYOUT', 'bins')


def default_fuse_dw():
    """Fuse depthwise 5x5 (stride 1) with the 1x1 conv that follows it into one kernel (k_dw_gemm)?  Off by default:
    the fused kernel is bit-identical to the two-kernel schedule, but one CTA per SM leaves only 8 depthwise warps per
    SM where the stand-alone depthwise kernel runs 16, the depthwise FMA loop is issue bound, and outputs wider than 192
    channels recompute the depthwise sums once per column block.  PIFPAF_FUSE_DW=1 turns it on."""
    return os.environ.get('PIFPAF_FUSE_DW', '0') == '1'


def _scatter_rows(wb, order, in_cols, k_cols):
    """GEMM operands of a 1x1 conv (w [n, c_in, ...], b [n]): weights [len(order), k_cols] whose row j is output channel
    order[j] (-1: a zero padding row) and whose column in_cols[i] holds input channel i, and the bias [len(order)]"""
    w, b = wb
    w = w.reshape(w.shape[0], -1)
    assert len(in_cols) == w.shape[1]
    real = order >= 0
    wp = np.zeros((len(order), k_cols), dtype=np.float32)
    wp[np.ix_(np.nonzero(real)[0], in_cols)] = w[order[real]]
    bp = np.zeros((len(order),), dtype=np.float32)
    bp[real] = b[order[real]]
    return wp, bp


def _dw_rows(wb, kernel, width, cols=None):
    """depthwise weights [width, kernel^2] and bias [width] with channel i of wb at row cols[i] (default: row i), zero
    elsewhere"""
    w, b = wb
    c = w.shape[0]
    cols = np.arange(c) if cols is None else cols
    wp = np.zeros((width, kernel * kernel), dtype=np.float32)
    bp = np.zeros((width,), dtype=np.float32)
    wp[cols] = w.reshape(c, kernel * kernel)
    bp[cols] = b
    return wp, bp


def conv_out_hw(h, w, kernel, stride, pad, dilation=1, ceil_mode=False):
    """Output size of a conv window (torch.nn.Conv2d / MaxPool2d) on an h x w input; a size < 1 means the window does
    not fit in the padded input.  ceil_mode: MaxPool2d(ceil_mode=True) -- the division rounds up, and a last window
    that would start at or beyond n + pad (in the right padding) is dropped.  The one rule the lowering and
    `tensor_shapes_at` size tensors by."""
    span = dilation * (kernel - 1) + 1

    def size(n):
        if not ceil_mode or n + 2 * pad < span:
            return (n + 2 * pad - span) // stride + 1
        out = (n + 2 * pad - span + stride - 1) // stride + 1
        return out - 1 if (out - 1) * stride >= n + pad else out
    return size(h), size(w)


def tensor_shapes_at(ops, capacity_shapes, in_h, in_w):
    """The tensors (h, w, c_phys) of a lowering (`build_ops` at its capacity: `capacity_shapes`, `ops`) at another input
    size, derived op by op with the rule `build_ops` lowered them with: what `build_ops(plan, in_h, in_w)` would give
    (for a heads-only plan in_h x in_w is the feature map).  Raises RuntimeError where an op's output would be empty or
    a tensor larger than its capacity in h or w."""
    shapes = [None] * len(capacity_shapes)

    def put(t, hw, op):
        if hw[0] < 1 or hw[1] < 1:
            raise RuntimeError(f'input {in_h}x{in_w}: the {op} op would have an empty output')
        if shapes[t] is not None and shapes[t] != hw:
            raise RuntimeError(f'tensor {t} gets two sizes, {shapes[t]} and {hw}')
        shapes[t] = hw

    for o in ops:
        kind = o['kind']
        if kind == 'input_conv':
            put(o['out'], conv_out_hw(in_h, in_w, o['kernel'], o['stride'], o['pad']), kind)
            continue
        if shapes[o['in']] is None:          # read before anything wrote it: the net's input (heads-only plans)
            shapes[o['in']] = (in_h, in_w)
        h, w = shapes[o['in']]
        if kind in ('conv', 'dwconv'):
            hw = conv_out_hw(h, w, o['kernel'], o['stride'], o['pad'], o.get('dilation', 1))
        elif kind == 'maxpool':
            hw = conv_out_hw(h, w, 3, o['stride'], 1, ceil_mode=o.get('ceil_mode', False))
        else:                               # 1x1 convs, the fused depthwise 5x5 (pad 2) -> 1x1, the heads
            hw = (h, w)
        outs = [pc[2] for pc in o['pieces']] if 'pieces' in o else [o[k] for k in ('out', 'residual', 'shuffle_src')
                                                                     if o.get(k, -1) >= 0]
        for t in outs:
            put(t, hw, kind)
    out = []
    for t, ((ch, cw, c), hw) in enumerate(zip(capacity_shapes, shapes)):
        if hw is None:
            hw = (in_h, in_w)
        if hw[0] > ch or hw[1] > cw:
            raise RuntimeError(f'input {in_h}x{in_w}: tensor {t} would be {hw[0]}x{hw[1]}, above its capacity {ch}x{cw}')
        out.append((hw[0], hw[1], c))
    return out


class _OpList:
    """The tensors (tensors[i] = (h, w, c_phys)) and ops of one lowering.  Each op kind is written by one method here,
    whose dict fields are the C ABI arguments (include/pifpaf_b200.h); the lowerings only wire them.  Methods without a
    t_out argument add their output tensor and return it."""

    def __init__(self):
        self.tensors, self.ops = [], []

    def tensor(self, h, w, c):
        self.tensors.append((h, w, c))
        return len(self.tensors) - 1

    def out_hw(self, t_in, e):
        """output size of the conv entry e (kernel, stride, pad, optional dilation) on tensor t_in"""
        h, w, _ = self.tensors[t_in]
        return conv_out_hw(h, w, e['kernel'], e['stride'], e['pad'], e.get('dilation', 1))

    def input_conv(self, inp, in_h, in_w, act):
        """the stem on the [3, in_h, in_w] image"""
        k, c = inp['w'].shape[-1], inp['w'].shape[0]
        t = self.tensor(*conv_out_hw(in_h, in_w, k, inp['stride'], inp['pad']), pad16(c))
        self.ops.append({'kind': 'input_conv', 'in_h': in_h, 'in_w': in_w, 'kernel': k, 'stride': inp['stride'],
                         'pad': inp['pad'], 'c_out': c, 'w': _f32(inp['w']), 'b': _f32(inp['b']), 'relu': act,
                         'out': t})
        return t

    def conv(self, t_in, e, act, residual=-1, out=None):
        """implicit-GEMM conv of entry e; residual: a tensor added to the output before the activation; out: (tensor,
        first column) of an existing tensor to write (default: a new tensor, from column 0)"""
        n = e['w'].shape[0]
        t, off = (self.tensor(*self.out_hw(t_in, e), pad16(n)), 0) if out is None else out
        self.ops.append({'kind': 'conv', 'in': t_in, 'in_off': 0, 'c_in': e['w'].shape[1], 'kernel': e['kernel'],
                         'stride': e['stride'], 'pad': e['pad'], 'dilation': e.get('dilation', 1), 'n_out': n,
                         'w': _f32(e['w']), 'b': _f32(e['b']), 'relu': int(act), 'out': t, 'out_off': int(off),
                         'residual': residual, 'residual_off': 0})
        return t

    def dwconv(self, t_in, wb, e, act=0, cols=None, width=None):
        """depthwise conv with the kernel, stride, pad and dilation of entry e.  cols: the channel of t_in each weight
        row meets (default: in order); width: the channels the op covers and the output's pitch (default: the weights'
        channels, the output padded to 16)"""
        c = wb[0].shape[0]
        t = self.tensor(*self.out_hw(t_in, e), pad16(c) if width is None else width)
        w, b = _dw_rows(wb, e['kernel'], c if width is None else width, cols)
        op = {'kind': 'dwconv', 'in': t_in, 'in_off': 0, 'channels': w.shape[0], 'kernel': e['kernel'],
              'stride': e['stride'], 'pad': e['pad'], 'w': w, 'b': b, 'relu': act, 'out': t, 'out_off': 0}
        if e.get('dilation', 1) != 1:
            op['dilation'] = e['dilation']
        self.ops.append(op)
        return t

    def conv1x1(self, t_in, in_off, in_cols, k_cols, wb, act, t_out, shuffle=None):
        """1x1 conv GEMM over k_cols columns of t_in from in_off (input channel i at column in_cols[i]); shuffle =
        (tensor, column): write the output interleaved with those pass-through channels (cat + channel_shuffle)"""
        n = wb[0].shape[0]
        w, b = _scatter_rows(wb, np.arange(n), in_cols, k_cols)
        s_t, s_off = (-1, 0) if shuffle is None else shuffle
        self.ops.append({'kind': 'conv1x1', 'in': t_in, 'in_off': in_off, 'k_cols': k_cols, 'n_out': n,
                         'w': w, 'b': b, 'relu': int(act), 'out': t_out, 'out_off': 0,
                         'shuffle_src': s_t, 'shuffle_off': s_off})

    def conv1x1_scatter(self, t_in, in_cols, k_cols, wb, act, order, pieces):
        """1x1 conv whose GEMM columns are the producer's output channels in `order` (-1: padding column, zero
        weights) and whose column pieces (col0, count, tensor, tensor_col) go to different tensors"""
        w, b = _scatter_rows(wb, order, in_cols, k_cols)
        self.ops.append({'kind': 'conv1x1', 'in': t_in, 'in_off': 0, 'k_cols': k_cols, 'n_out': len(order),
                         'w': w, 'b': b, 'relu': int(act), 'out': pieces[0][2], 'out_off': pieces[0][3],
                         'shuffle_src': -1, 'shuffle_off': 0, 'pieces': [tuple(int(v) for v in pc) for pc in pieces]})

    def dw_conv1x1_scatter(self, t_in, width, dw_wb, e, wb, act, order, pieces):
        """the depthwise conv of entry e on the first len(dw) of `width` channels of t_in, then conv1x1_scatter on its
        output -- one fused kernel, no intermediate tensor"""
        dw_w, dw_b = _dw_rows(dw_wb, e['kernel'], width)
        w, b = _scatter_rows(wb, order, np.arange(dw_wb[0].shape[0]), width)
        self.ops.append({'kind': 'dw_conv1x1', 'in': t_in, 'in_off': 0, 'channels': width, 'kernel': e['kernel'],
                         'stride': e['stride'], 'pad': e['pad'], 'dw_w': dw_w, 'dw_b': dw_b, 'dw_relu': 0,
                         'n_out': len(order), 'w': w, 'b': b, 'relu': int(act), 'out': pieces[0][2],
                         'pieces': [tuple(int(v) for v in pc) for pc in pieces]})

    def maxpool(self, t_in, channels, stride, ceil_mode=False):
        """3x3 max pool, padding 1; 'ceil_mode' only where it is set"""
        h, w, _ = self.tensors[t_in]
        t = self.tensor(*conv_out_hw(h, w, 3, stride, 1, ceil_mode=ceil_mode), pad16(channels))
        op = {'kind': 'maxpool', 'in': t_in, 'in_off': 0, 'channels': channels, 'stride': stride, 'out': t, 'out_off': 0}
        if ceil_mode:
            op['ceil_mode'] = True
        self.ops.append(op)
        return t

    def heads(self, heads, t_in, k_cols, cols=None):
        """all heads as one GEMM with the CompositeField4 eval epilogue; cols: the physical column of each logical input
        channel (None: column c holds channel c)"""
        w = _f32(np.concatenate([_f32(hd['w']) for hd in heads], axis=0))
        if cols is not None:
            wp = np.zeros((w.shape[0], k_cols), dtype=np.float32)
            wp[:, cols] = w
            w = wp
        self.ops.append({'kind': 'heads', 'in': t_in, 'k_cols': k_cols, 'upsample': int(heads[0].get('upsample', 1)),
                         'n_fields': [hd['n_fields'] for hd in heads], 'n_comp': [hd['n_comp'] for hd in heads],
                         'ops': [o for hd in heads for o in hd['ops']], 'w': w,
                         'b': _f32(np.concatenate([_f32(hd['b']) for hd in heads], axis=0))})


def build_ops(plan, in_h, in_w, layout=None, fuse_dw=None):
    """Lower a plan to the op list of libpifpaf_b200 (pure Python; no GPU needed).  layout and fuse_dw apply to
    ShuffleNetV2K plans (default_layout, default_fuse_dw) and are ignored for the others.

    Returns (tensors, ops, info): tensors[i] = (h, w, c_phys); ops are dicts with a 'kind' in
    {'input_conv', 'conv1x1', 'dwconv', 'dw_conv1x1', 'conv', 'maxpool', 'heads'} whose fields are the C ABI
    arguments (written by _OpList); info = {'block_outputs': [(tensor, _Layout)], 'feature': (tensor, _Layout)}."""
    L = _OpList()
    kind = plan.get('kind')
    if kind == 'shufflenetv2k':
        info = _lower_shufflenetv2k(L, plan, in_h, in_w, layout, fuse_dw)
    elif kind == 'resnet':
        info = _lower_resnet(L, plan, in_h, in_w)
    elif kind == 'mobilenetv2':
        info = _lower_mobilenetv2(L, plan, in_h, in_w)
    elif kind == 'squeezenet':
        info = _lower_squeezenet(L, plan, in_h, in_w)
    elif kind == 'heads_only':
        # in_h x in_w is the FEATURE map here; the feature tensor is filled through CompiledNet.forward_features
        c_in = int(plan['c_in'])
        L.heads(plan['heads'], L.tensor(in_h, in_w, pad16(c_in)), c_in)
        info = {'block_outputs': [], 'feature': (0, _Layout(c_in, split=False))}
    else:
        raise RuntimeError('unsupported plan kind')
    return L.tensors, L.ops, info


def _lower_shufflenetv2k(L, plan, in_h, in_w, layout, fuse_dw):
    layout = default_layout() if layout is None else layout
    if layout not in ('bins', 'shuffle'):
        raise RuntimeError("layout must be 'bins' or 'shuffle'")
    fuse_dw = default_fuse_dw() if fuse_dw is None else bool(fuse_dw)
    tensor = L.tensor
    cur = L.input_conv(plan['input'], in_h, in_w, ACT_RELU)
    if plan.get('input2') is not None:
        # --shufflenetv2k-input-conv2-stride: 3x3 conv + BN + ReLU on the stem output (basenetworks.py:283-294), an
        # implicit-GEMM conv op
        cur = L.conv(cur, plan['input2'], ACT_RELU)
    h, w, _ = L.tensors[cur]
    lay = _Layout((plan.get('input2') or plan['input'])['w'].shape[0], split=False)
    stages = list(plan['stages'])
    if plan.get('conv5_stage') is not None:
        # --shufflenetv2k-conv5-as-stage: without a branch1 (stage 4 as wide as conv5) the two blocks continue stage 4
        # (same width, same dilation), otherwise they are one more stage whose first block has stride 1
        c5s = plan['conv5_stage']
        stages = stages[:-1] + [stages[-1] + c5s] if not c5s[0]['first'] else stages + [c5s]
    block_outputs = []
    for blocks in stages if layout == 'bins' else []:
        # ---- 'bins' layout: every channel is written once, into the buffer of the block that consumes it
        bf = blocks[0]['b2_pw2'][0].shape[0]
        hp = _branch_pitch(bf)
        e0 = blocks[0]
        ho, wo = L.out_hw(cur, e0)
        producers, bins, final = _plan_stage_bins(bf, len(blocks))
        t_bin = {t: tensor(ho, wo, pad16(bins[t]['width'])) for t in bins}
        t_bin['final'] = tensor(ho, wo, pad16(final['width']))

        def pieces_of(k):
            return [(c0_, cnt, t_bin[d], dc) for (c0_, cnt, d, dc) in producers[k]['pieces']]

        cols = lay.cols()
        # block 0, branch1: dw (stride) -> 1x1; branch2: 1x1 -> dw (stride) -> 1x1   (basenetworks.py:200-226)
        t_a = L.dwconv(cur, e0['b1_dw'], e0, cols=cols, width=lay.width)
        L.conv1x1_scatter(t_a, cols, lay.width, e0['b1_pw'], True, producers[0]['order'], pieces_of(0))
        # the tensor in front of the STRIDE-2 depthwise conv gets 128-byte pixels (_dw_in_pitch).  Its producer leaves the padding
        # channels unwritten (rows with a 32-byte hole) and does not pay for writing them.
        t_c = tensor(h, w, _dw_in_pitch(bf))
        L.conv1x1(cur, 0, cols, lay.width, e0['b2_pw1'], True, t_c)
        t_d = L.dwconv(t_c, e0['b2_dw'], e0, width=hp)
        L.conv1x1_scatter(t_d, np.arange(bf), hp, e0['b2_pw2'], True, producers[1]['order'], pieces_of(1))
        h, w = ho, wo
        for t, e in enumerate(blocks[1:], start=1):
            assert not e['first'] and e['stride'] == 1 and e['b2_pw2'][0].shape[0] == bf
            # x2 = the bin of block t: slot j holds the channel that meets weight column wcol[j] of the first 1x1
            wcol = bins[t]['wcol']
            in_cols = np.empty((bf,), dtype=np.int64)
            in_cols[wcol[wcol >= 0]] = np.nonzero(wcol >= 0)[0]
            t_c = tensor(h, w, hp)          # stride-1 depthwise launches are issue bound: the padding buys nothing there
            L.conv1x1(t_bin[t], 0, in_cols, L.tensors[t_bin[t]][2], e['b2_pw1'], True, t_c)
            order = producers[t + 1]['order']
            # k_dw_gemm is built for the undilated 5x5, pad 2
            if fuse_dw and e['kernel'] == 5 and e['pad'] == 2 and e.get('dilation', 1) == 1 and len(order) <= 512:
                L.dw_conv1x1_scatter(t_c, hp, e['b2_dw'], e, e['b2_pw2'], True, order, pieces_of(t + 1))
                continue
            t_d = L.dwconv(t_c, e['b2_dw'], e, width=hp)
            L.conv1x1_scatter(t_d, np.arange(bf), hp, e['b2_pw2'], True, order, pieces_of(t + 1))
        logical = final['logical']
        phys = np.empty((2 * bf,), dtype=np.int64)
        phys[logical[logical >= 0]] = np.nonzero(logical >= 0)[0]
        cur, lay = t_bin['final'], _Layout(2 * bf, split=False, phys=phys, width=L.tensors[t_bin['final']][2])
        block_outputs.append((cur, lay))
    for blocks in stages if layout == 'shuffle' else []:
        for e in blocks:
            bf = e['b2_pw2'][0].shape[0]
            hp = pad16(bf)
            ho, wo = L.out_hw(cur, e)
            out_lay = _Layout(2 * bf, split=True)
            t_out = tensor(ho, wo, out_lay.width)
            if e['first']:
                cols = lay.cols()
                # branch1: dw (stride) -> 1x1   (basenetworks.py:200-212)
                t_a = L.dwconv(cur, e['b1_dw'], e, cols=cols, width=lay.width)
                t_b = tensor(ho, wo, hp)
                L.conv1x1(t_a, 0, cols, lay.width, e['b1_pw'], True, t_b)
                # branch2: 1x1 -> dw (stride) -> 1x1   (basenetworks.py:214-226)
                t_c = tensor(h, w, hp)
                L.conv1x1(cur, 0, cols, lay.width, e['b2_pw1'], True, t_c)
                t_d = L.dwconv(t_c, e['b2_dw'], e, width=hp)
                L.conv1x1(t_d, 0, np.arange(bf), hp, e['b2_pw2'], True, t_out, shuffle=(t_b, 0))
            else:
                assert lay.split and lay.half == bf
                # x1, x2 = x.chunk(2): x2 is the column window [bf, 2*bf) (basenetworks.py:234-236).  TMA needs a
                # 16-byte aligned start (32 bytes or more is faster), so the view begins at _view_start(bf) <= bf;
                # the leading columns are pass-through channels and get zero weights.
                a0 = _view_start(bf)
                lead = bf - a0
                t_c = tensor(h, w, hp)
                L.conv1x1(cur, a0, lead + np.arange(bf), lead + bf, e['b2_pw1'], True, t_c)
                t_d = L.dwconv(t_c, e['b2_dw'], e, width=hp)
                L.conv1x1(t_d, 0, np.arange(bf), hp, e['b2_pw2'], True, t_out, shuffle=(cur, 0))
            cur, lay, h, w = t_out, out_lay, ho, wo
            block_outputs.append((cur, lay))
    if plan.get('conv5_stage') is not None:
        # the heads read the last stage output as it lies: lay.width columns in physical order
        L.heads(plan['heads'], cur, lay.width, lay.cols())
        return {'block_outputs': block_outputs, 'feature': (cur, lay)}
    c5 = plan['conv5'][0].shape[0]
    t5 = tensor(h, w, pad16(c5))
    L.conv1x1(cur, 0, lay.cols(), lay.width, plan['conv5'], True, t5)
    L.heads(plan['heads'], t5, c5)
    return {'block_outputs': block_outputs, 'feature': (t5, _Layout(c5, split=False))}


def _lower_resnet(L, plan, in_h, in_w):
    """torchvision BasicBlock / Bottleneck (eval): every conv+BN is one implicit-GEMM conv op; the residual
    add and the final ReLU of a block are fused into the epilogue of its last conv."""
    cur = L.input_conv(plan['input'], in_h, in_w, ACT_RELU)
    if plan.get('pool') is not None:
        cur = L.maxpool(cur, plan['input']['w'].shape[0], plan['pool']['stride'])
    if plan.get('input2') is not None:
        cur = L.conv(cur, plan['input2'], ACT_RELU)
    block_outputs = []
    for e in plan['blocks']:
        identity = cur if e['downsample'] is None else L.conv(cur, e['downsample'], ACT_NONE)
        for i, ce in enumerate(e['convs']):
            cur = L.conv(cur, ce, ACT_RELU, residual=identity if i == len(e['convs']) - 1 else -1)
        block_outputs.append((cur, _Layout(e['convs'][-1]['w'].shape[0], split=False)))
    c = plan['blocks'][-1]['convs'][-1]['w'].shape[0]
    L.heads(plan['heads'], cur, c)
    return {'block_outputs': block_outputs, 'feature': (cur, _Layout(c, split=False))}


def _lower_mobilenetv2(L, plan, in_h, in_w):
    """torchvision InvertedResidual (eval): the expand 1x1 and the linear projection are implicit-GEMM conv ops (the
    projection adds the block input in its epilogue), the 3x3 depthwise conv a dwconv op; every activation is ReLU6.
    Tensors are padded to 16 channels (24 -> 32)."""
    cur = L.input_conv(plan['input'], in_h, in_w, ACT_RELU6)
    block_outputs = []
    for e in plan['blocks']:
        x = cur
        if e['expand'] is not None:
            cur = L.conv(cur, e['expand'], ACT_RELU6)
        cur = L.dwconv(cur, (e['dw']['w'], e['dw']['b']), e['dw'], ACT_RELU6)
        cur = L.conv(cur, e['project'], ACT_NONE, residual=x if e['residual'] else -1)
        block_outputs.append((cur, _Layout(e['project']['w'].shape[0], split=False)))
    c = plan['last']['w'].shape[0]
    cur = L.conv(cur, plan['last'], ACT_RELU6)
    L.heads(plan['heads'], cur, c)
    return {'block_outputs': block_outputs, 'feature': (cur, _Layout(c, split=False))}


def _lower_squeezenet(L, plan, in_h, in_w):
    """torchvision SqueezeNet 1.1 features (eval): the stem and every Fire conv are implicit-GEMM conv ops with ReLU, the
    pools ceil-mode max pool ops.  A Fire's two expand convs read its squeeze output and write columns [0, e1) and
    [e1, e1 + e3) of one tensor, so torch.cat never runs."""
    cur = L.input_conv(plan['input'], in_h, in_w, ACT_RELU)
    c = plan['input']['w'].shape[0]
    block_outputs = []
    for layer in plan['layers']:
        if layer['type'] == 'pool':
            cur = L.maxpool(cur, c, layer['stride'], ceil_mode=layer['ceil_mode'])
            continue
        sq = L.conv(cur, layer['squeeze'], ACT_RELU)
        e1, e3 = layer['expand1x1'], layer['expand3x3']
        n1 = e1['w'].shape[0]
        c = n1 + e3['w'].shape[0]
        cur = L.tensor(*L.out_hw(sq, e1), pad16(c))
        L.conv(sq, e1, ACT_RELU, out=(cur, 0))
        L.conv(sq, e3, ACT_RELU, out=(cur, n1))
        block_outputs.append((cur, _Layout(c, split=False)))
    L.heads(plan['heads'], cur, c)
    return {'block_outputs': block_outputs, 'feature': (cur, _Layout(c, split=False))}


class CompiledNet:
    """A plan compiled to libpifpaf_b200 ops for a maximum input size and batch.  in_h, in_w is that capacity; the net
    runs at any input size up to it (`set_input_size`), each tensor packed densely in the buffer allocated for the
    capacity, and computes there what a net compiled at exactly that size computes."""

    def __init__(self, plan, in_h, in_w, max_batch, device=0, layout=None, fuse_dw=None):
        self.lib = _lib.lib()
        self.device = int(device)
        self.max_batch = int(max_batch)
        self.in_h, self.in_w = int(in_h), int(in_w)
        self.tensor_shapes, ops, self.info = build_ops(plan, self.in_h, self.in_w, layout=layout, fuse_dw=fuse_dw)
        self.capacity_shapes = list(self.tensor_shapes)
        self._input_size = (self.in_h, self.in_w)
        self.op_desc = [{k: v for k, v in o.items() if not isinstance(v, np.ndarray)} for o in ops]
        self.handle = ctypes.c_void_p()
        _lib.check(self.lib.pifpaf_net_create(ctypes.byref(self.handle), self.device, self.max_batch))
        self._emit(ops)
        self.flops_per_image = float(self.lib.pifpaf_net_flops_per_image(self.handle))
        self.num_ops = int(self.lib.pifpaf_net_num_ops(self.handle))
        self.heads = []
        for i, h in enumerate(plan['heads']):
            ptr = ctypes.c_void_p()
            nf, nc, hh, ww = (ctypes.c_int32() for _ in range(4))
            _lib.check(self.lib.pifpaf_net_head_output(self.handle, i, ctypes.byref(ptr), ctypes.byref(nf),
                                                       ctypes.byref(nc), ctypes.byref(hh), ctypes.byref(ww)))
            self.heads.append({'ptr': ptr.value, 'n_fields': nf.value, 'n_comp': nc.value,
                               'h': hh.value, 'w': ww.value, 'stride': h['stride']})

    @property
    def input_size(self):
        """(h, w) the forwards take now: the capacity (in_h, in_w) until `set_input_size` changes it."""
        return self._input_size

    def set_input_size(self, h, w):
        """Run the following forwards on [B, 3, h, w] images (for a heads-only plan: h x w feature maps).  The tensors
        and head outputs take the sizes a net compiled at h x w has (`tensor_shapes`, heads[i]['h'], ['w']); taps and
        head views cover that size.  A size above the capacity in any tensor, or one that empties a layer, raises
        RuntimeError and leaves the previous size in force.  A forward still running keeps its own size; the head
        outputs it writes are reused by the next forward as before."""
        h, w = int(h), int(w)
        if (h, w) == self._input_size:
            return
        if not (1 <= h <= self.in_h and 1 <= w <= self.in_w):
            raise RuntimeError(f'input size {h}x{w}: outside 1x1 .. the capacity {self.in_h}x{self.in_w}')
        shapes = tensor_shapes_at(self.op_desc, self.capacity_shapes, h, w)
        table = np.ascontiguousarray([hw for s in shapes for hw in s[:2]], dtype=np.int32)
        _lib.check(self.lib.pifpaf_net_set_input_size(self.handle, h, w, len(shapes), _ptr(table)))
        self.tensor_shapes, self._input_size = shapes, (h, w)
        self.flops_per_image = float(self.lib.pifpaf_net_flops_per_image(self.handle))
        for i, hd in enumerate(self.heads):
            hh, ww = ctypes.c_int32(), ctypes.c_int32()
            _lib.check(self.lib.pifpaf_net_head_output(self.handle, i, None, None, None, ctypes.byref(hh),
                                                       ctypes.byref(ww)))
            hd['h'], hd['w'] = hh.value, ww.value

    def __del__(self):
        self.close()

    def close(self):
        """Free every device buffer of the net (idempotent)."""
        h, self.handle = getattr(self, 'handle', None), None
        if h:
            try:
                self.lib.pifpaf_net_destroy(h)
            except Exception:
                pass

    def set_head_buffers(self, n):
        """1: head outputs are valid until the next forward (default); 2: successive forwards alternate between two
        sets, so a decode of forward i may run concurrently with forward i+1."""
        _lib.check(self.lib.pifpaf_net_set_head_buffers(self.handle, int(n)))

    def set_sm_limit(self, n_sm):
        """Cap the persistent grids of the forward at n_sm SMs (0: all of them)."""
        _lib.check(self.lib.pifpaf_net_set_sm_limit(self.handle, int(n_sm)))

    def _emit(self, ops):
        L, H = self.lib, self.handle
        for (h, w, c) in self.tensor_shapes:
            tid = ctypes.c_int32(-1)
            _lib.check(L.pifpaf_net_tensor(H, h, w, c, ctypes.byref(tid)))
        for o in ops:
            if o['kind'] == 'input_conv':
                _lib.check(L.pifpaf_net_input_conv(H, o['in_h'], o['in_w'], o['kernel'], o['stride'], o['pad'],
                                                   o['c_out'], _ptr(o['w']), _ptr(o['b']), o['relu'], o['out']))
            elif o['kind'] == 'dw_conv1x1':
                pcs = np.ascontiguousarray(np.asarray(o['pieces'], dtype=np.int32).T)
                _lib.check(L.pifpaf_net_dw_conv1x1_scatter(
                    H, o['in'], o['in_off'], o['channels'], o['kernel'], o['stride'], o['pad'], _ptr(o['dw_w']),
                    _ptr(o['dw_b']), o['dw_relu'], o['n_out'], _ptr(o['w']), _ptr(o['b']), o['relu'], pcs.shape[1],
                    _ptr(pcs[0]), _ptr(pcs[1]), _ptr(pcs[2]), _ptr(pcs[3])))
            elif o['kind'] == 'conv1x1' and 'pieces' in o:
                pcs = np.ascontiguousarray(np.asarray(o['pieces'], dtype=np.int32).T)     # rows: col0, count, tensor, col
                _lib.check(L.pifpaf_net_conv1x1_scatter(H, o['in'], o['in_off'], o['k_cols'], o['n_out'],
                                                        _ptr(o['w']), _ptr(o['b']), o['relu'], pcs.shape[1],
                                                        _ptr(pcs[0]), _ptr(pcs[1]), _ptr(pcs[2]), _ptr(pcs[3])))
            elif o['kind'] == 'conv1x1':
                _lib.check(L.pifpaf_net_conv1x1(H, o['in'], o['in_off'], o['k_cols'], o['n_out'], _ptr(o['w']),
                                                _ptr(o['b']), o['relu'], o['out'], o['out_off'],
                                                o['shuffle_src'], o['shuffle_off']))
            elif o['kind'] == 'conv':
                _lib.check(L.pifpaf_net_conv_dilated(H, o['in'], o['in_off'], o['c_in'], o['kernel'], o['stride'],
                                                     o['pad'], o['n_out'], _ptr(o['w']), _ptr(o['b']), o['relu'],
                                                     o['out'], o['out_off'], o['residual'], o['residual_off'],
                                                     o['dilation']))
            elif o['kind'] == 'maxpool':
                _lib.check(L.pifpaf_net_maxpool_ceil(H, o['in'], o['in_off'], o['channels'], o['stride'], o['out'],
                                                     o['out_off'], int(o.get('ceil_mode', False))))
            elif o['kind'] == 'dwconv':
                _lib.check(L.pifpaf_net_dwconv_dilated(H, o['in'], o['in_off'], o['channels'], o['kernel'],
                                                       o['stride'], o['pad'], _ptr(o['w']), _ptr(o['b']), o['relu'],
                                                       o['out'], o['out_off'], o.get('dilation', 1)))
            elif o['kind'] == 'heads':
                n = len(o['n_fields'])
                nf = (ctypes.c_int32 * n)(*o['n_fields'])
                nc = (ctypes.c_int32 * n)(*o['n_comp'])
                ops_c = (ctypes.c_int32 * len(o['ops']))(*o['ops'])
                _lib.check(L.pifpaf_net_heads_upsampled(H, o['in'], o['k_cols'], n, nf, nc, ops_c, int(o.get('upsample', 1)),
                                                        _ptr(o['w']), _ptr(o['b'])))
            else:
                raise RuntimeError(o['kind'])

    # --- execution -----------------------------------------------------------
    def forward(self, image_batch, *, gemm_impl=0, stream=None):
        """Shell.forward: image_batch [B,3,H,W] float32 CUDA -> tuple of [B,F,comp,h,w] float32 CUDA views
        (valid until the next forward)."""
        if not image_batch.is_cuda or image_batch.dtype != torch.float32:
            raise RuntimeError('image_batch must be a float32 CUDA tensor')
        if image_batch.dim() != 4 or image_batch.shape[1] != 3 or tuple(image_batch.shape[2:]) != self._input_size:
            raise RuntimeError('expected [B,3,{},{}]'.format(*self._input_size))
        b = int(image_batch.shape[0])
        if b > self.max_batch:
            raise RuntimeError('batch exceeds max_batch')
        image_batch = image_batch.contiguous()
        st = stream if stream is not None else torch.cuda.current_stream(image_batch.device)
        _lib.check(self.lib.pifpaf_net_forward(self.handle, image_batch.data_ptr(), b, int(gemm_impl),
                                               ctypes.c_void_p(st.cuda_stream)))
        self._keepalive = image_batch
        return self._head_views(b)

    def _head_views(self, b):
        outs = []
        for i, hd in enumerate(self.heads):
            ptr = ctypes.c_void_p()       # the buffer set the last forward wrote (set_head_buffers)
            _lib.check(self.lib.pifpaf_net_head_output(self.handle, i, ctypes.byref(ptr), None, None, None, None))
            arr = _DevArray(ptr.value, (b, hd['n_fields'], hd['n_comp'], hd['h'], hd['w']))
            outs.append(torch.as_tensor(arr, device=f'cuda:{self.device}'))
        return tuple(outs)

    def forward_features(self, features, *, gemm_impl=0, stream=None):
        """CompositeField4 heads alone (heads.py:330-378) on a given feature map: features [B,h,w,C] float32
        (host numpy or tensor; rounded to bf16 on upload) -> head outputs.  For plans of kind 'heads_only'
        (`heads_only_plan`): parity / accuracy tests feed the heads GEMM with controlled activations."""
        if self.op_desc[0]['kind'] != 'heads':
            raise RuntimeError('forward_features needs a heads_only plan')
        f = np.ascontiguousarray(features.cpu().numpy() if isinstance(features, torch.Tensor) else features,
                                 dtype=np.float32)
        b = int(f.shape[0])
        h, w, c = self.tensor_shapes[0]
        if f.shape[1:3] != (h, w) or f.shape[3] > c or b > self.max_batch:
            raise RuntimeError(f'expected features [B<={self.max_batch},{h},{w},<={c}]')
        padded = np.zeros((b, h, w, c), dtype=np.float32)
        padded[..., :f.shape[3]] = f
        _lib.check(self.lib.pifpaf_net_set_tensor(self.handle, 0, b, _ptr(padded), padded.size))
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        _lib.check(self.lib.pifpaf_net_forward(self.handle, None, b, int(gemm_impl), ctypes.c_void_p(st.cuda_stream)))
        return self._head_views(b)

    # the reference's eval preprocessing constants (transforms/__init__.py:26-33)
    IMAGE_MEAN = (0.485, 0.456, 0.406)
    IMAGE_STD = (0.229, 0.224, 0.225)

    def forward_uint8(self, image_batch, *, mean=IMAGE_MEAN, std=IMAGE_STD, gemm_impl=0, stream=None):
        """Shell.forward on raw images: image_batch [B,H,W,3] uint8 CUDA (HWC, as PIL / numpy hold them).  ToTensor
        and Normalize(mean, std) of the reference's EVAL_TRANSFORM are applied inside the stem kernel; the result
        equals forward() on the normalised float batch bit for bit."""
        if not image_batch.is_cuda or image_batch.dtype != torch.uint8:
            raise RuntimeError('image_batch must be a uint8 CUDA tensor')
        if image_batch.dim() != 4 or image_batch.shape[3] != 3 or tuple(image_batch.shape[1:3]) != self._input_size:
            raise RuntimeError('expected [B,{},{},3]'.format(*self._input_size))
        b = int(image_batch.shape[0])
        if b > self.max_batch:
            raise RuntimeError('batch exceeds max_batch')
        image_batch = image_batch.contiguous()
        st = stream if stream is not None else torch.cuda.current_stream(image_batch.device)
        m = (ctypes.c_float * 3)(*[float(v) for v in mean])
        s = (ctypes.c_float * 3)(*[float(v) for v in std])
        _lib.check(self.lib.pifpaf_net_forward_u8(self.handle, image_batch.data_ptr(), b, m, s, int(gemm_impl),
                                                  ctypes.c_void_p(st.cuda_stream)))
        self._keepalive = image_batch
        return self._head_views(b)

    def forward_timed(self, image_batch, *, gemm_impl=0):
        """Profiling pass: per-op (ms, kind, flops, bytes); kind 0 input conv, 1 wgmma GEMM, 2 depthwise,
        3 fused kernels (depthwise -> GEMM, or 1x1 GEMM -> stride-2 depthwise: there the GEMM op launches nothing and
        reports 0 FLOPs and 0 bytes, and the depthwise op reports the fused launch with the FLOPs of both), 4 max pool."""
        b, n = int(image_batch.shape[0]), self.num_ops
        ms = np.zeros((n,), dtype=np.float32)
        kind = np.zeros((n,), dtype=np.int32)
        flops = np.zeros((n,), dtype=np.float64)
        nbytes = np.zeros((n,), dtype=np.float64)
        st = torch.cuda.current_stream(image_batch.device)
        _lib.check(self.lib.pifpaf_net_forward_timed(self.handle, image_batch.contiguous().data_ptr(), b,
                                                     int(gemm_impl), ctypes.c_void_p(st.cuda_stream),
                                                     _ptr(ms), _ptr(kind), _ptr(flops), _ptr(nbytes)))
        return ms, kind, flops, nbytes

    def tap(self, tensor_id, batch):
        """Debug: activation tensor as float32 numpy [B,h,w,c_phys].  A 1x1 output that the last forward kept
        inside the fused 1x1 -> depthwise kernel is computed first (its GEMM runs again at that forward's batch), so
        the tap returns what the two-kernel schedule writes."""
        h, w, c = self.tensor_shapes[tensor_id]
        out = np.empty((batch, h, w, c), dtype=np.float32)
        _lib.check(self.lib.pifpaf_net_tap_tensor(self.handle, tensor_id, batch, _ptr(out), out.size))
        return out
