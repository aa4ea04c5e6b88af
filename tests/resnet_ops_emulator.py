"""CPU (torch fp32) interpreter of the op list that openpifpaf_b200.network.build_ops emits for Resnet plans: the
stem, implicit-GEMM convs with dilation, the 3x3 max pool and the heads with upsample_stride (PixelShuffle + crop),
executed as include/pifpaf_b200.h documents them.  Test infrastructure, like tests/ops_emulator.py (which covers the
ShuffleNetV2K ops)."""
import math

import torch
import torch.nn.functional as F


def run_ops(tensors, ops, images, bf16=False):
    """images [B,3,H,W] float32 -> (list of head outputs [B,F,comp,h,w], activations [B,h,w,c_phys]).
    With ``bf16`` activations and the conv / head weights are rounded to bf16 where the kernels round them (the stem
    weights stay f32)."""
    B = images.shape[0]
    acts = [torch.zeros((B, h, w, c), dtype=torch.float32) for (h, w, c) in tensors]

    def q(x):
        return x.to(torch.bfloat16).to(torch.float32) if bf16 else x

    def nchw(o, c):
        return acts[o['in']][..., o['in_off']:o['in_off'] + c].permute(0, 3, 1, 2)

    heads_out = None
    for o in ops:
        kind = o['kind']
        if kind == 'input_conv':
            y = F.relu(F.conv2d(images, torch.from_numpy(o['w']), torch.from_numpy(o['b']), o['stride'], o['pad']))
            acts[o['out']][..., :o['c_out']] = q(y.permute(0, 2, 3, 1))
        elif kind == 'maxpool':
            y = F.max_pool2d(nchw(o, o['channels']), 3, o['stride'], 1)
            acts[o['out']][..., o['out_off']:o['out_off'] + o['channels']] = y.permute(0, 2, 3, 1)
        elif kind == 'conv':
            y = F.conv2d(nchw(o, o['c_in']), q(torch.from_numpy(o['w'])), torch.from_numpy(o['b']), o['stride'], o['pad'],
                         o['dilation']).permute(0, 2, 3, 1)
            if o['residual'] >= 0:
                y = y + acts[o['residual']][..., o['residual_off']:o['residual_off'] + o['n_out']]
            if o['relu']:
                y = F.relu(y)
            acts[o['out']][..., o['out_off']:o['out_off'] + o['n_out']] = q(y)
        elif kind == 'heads':
            up = o['upsample']
            y = acts[o['in']][..., :o['k_cols']] @ q(torch.from_numpy(o['w'])).t() + torch.from_numpy(o['b'])
            heads_out, col, op_off = [], 0, 0
            for nf, nc in zip(o['n_fields'], o['n_comp']):
                t = y[..., col * up * up:(col + nf * nc) * up * up].permute(0, 3, 1, 2)
                if up > 1:
                    lo, hi = (up - 1) // 2, math.ceil((up - 1) / 2)
                    t = F.pixel_shuffle(t, up)
                    t = t[:, :, lo:t.shape[2] - hi, lo:t.shape[3] - hi]
                _, _, h, w = t.shape
                t = t.reshape(B, nf, nc, h, w).clone()
                for c_i in range(nc):
                    op = o['ops'][op_off + c_i]
                    if op == 1:
                        t[:, :, c_i] = torch.sigmoid(t[:, :, c_i])
                    elif op == 2:
                        t[:, :, c_i] += torch.arange(w, dtype=torch.float32)
                    elif op == 3:
                        t[:, :, c_i] += torch.arange(h, dtype=torch.float32).view(h, 1)
                    elif op == 4:
                        t[:, :, c_i] = F.softplus(t[:, :, c_i])
                heads_out.append(t)
                col += nf * nc
                op_off += nc
        else:
            raise ValueError(kind)
    return heads_out, acts
