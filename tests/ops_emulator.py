"""CPU (torch fp32) interpreter of the op list emitted by openpifpaf_b200.network.build_ops.

Test infrastructure: validates the host-side lowering (BN folding, physical channel
placement, fused cat+channel_shuffle, head epilogue ops) without a GPU by executing the
ops exactly as the C ABI documents them (include/pifpaf_b200.h) and comparing with the
oracle network.  Every op kind and field build_ops emits is covered: activation codes, conv
and depthwise dilation, the max pool, upsampled heads, scatter pieces and the fused
depthwise -> 1x1 op."""
import math

import torch
import torch.nn.functional as F


def act(y, code):
    """activation codes of include/pifpaf_b200.h: 0 none, 1 ReLU, 2 ReLU6"""
    if code == 1:
        return F.relu(y)
    if code == 2:
        return torch.clamp(y, 0.0, 6.0)
    assert code == 0, code
    return y


def run_ops(tensors, ops, images, bf16=False):
    """images [B,3,H,W] float32 -> (list of head outputs [B,F,comp,h,w], activations [B,h,w,c_phys]).

    With ``bf16`` activations and the weights of the GEMM-like ops (1x1, implicit-GEMM conv, heads) are rounded to bf16;
    depthwise and stem weights stay f32, as the kernels read them."""
    B = images.shape[0]
    acts = [torch.zeros((B, h, w, c), dtype=torch.float32) for (h, w, c) in tensors]

    def q(x):
        return x.to(torch.bfloat16).to(torch.float32) if bf16 else x

    def nchw(o, c):
        return acts[o['in']][..., o['in_off']:o['in_off'] + c].permute(0, 3, 1, 2)

    def scatter(o, y):
        for (c0, cnt, t_id, t_col) in o['pieces']:
            acts[t_id][..., t_col:t_col + cnt] = y[..., c0:c0 + cnt]

    heads_out = None
    for o in ops:
        kind = o['kind']
        if kind == 'input_conv':
            y = F.conv2d(images, torch.from_numpy(o['w']), torch.from_numpy(o['b']), o['stride'], o['pad'])
            acts[o['out']][..., :o['c_out']] = q(act(y, o['relu']).permute(0, 2, 3, 1))
        elif kind == 'conv1x1':
            a = acts[o['in']][..., o['in_off']:o['in_off'] + o['k_cols']]
            y = q(act(a @ q(torch.from_numpy(o['w'])).t() + torch.from_numpy(o['b']), o['relu']))
            n = o['n_out']
            out = acts[o['out']]
            if 'pieces' in o:
                scatter(o, y)
            elif o['shuffle_src'] < 0:
                out[..., o['out_off']:o['out_off'] + n] = y
            else:
                out[..., 0:2 * n:2] = acts[o['shuffle_src']][..., o['shuffle_off']:o['shuffle_off'] + n]
                out[..., 1:2 * n:2] = y
        elif kind == 'conv':
            y = F.conv2d(nchw(o, o['c_in']), q(torch.from_numpy(o['w'])), torch.from_numpy(o['b']), o['stride'],
                         o['pad'], o['dilation']).permute(0, 2, 3, 1)
            if o['residual'] >= 0:
                y = y + acts[o['residual']][..., o['residual_off']:o['residual_off'] + o['n_out']]
            acts[o['out']][..., o['out_off']:o['out_off'] + o['n_out']] = q(act(y, o['relu']))
        elif kind == 'dw_conv1x1':
            c, k = o['channels'], o['kernel']
            wdw = torch.from_numpy(o['dw_w']).reshape(c, 1, k, k)
            y = act(F.conv2d(nchw(o, c), wdw, torch.from_numpy(o['dw_b']), o['stride'], o['pad'], groups=c), o['dw_relu'])
            y = q(y.permute(0, 2, 3, 1))                    # the bf16 A operand of the fused GEMM
            scatter(o, q(act(y @ q(torch.from_numpy(o['w'])).t() + torch.from_numpy(o['b']), o['relu'])))
        elif kind == 'dwconv':
            c, k, d = o['channels'], o['kernel'], o.get('dilation', 1)
            # a dilated kernel as the equivalent (k - 1) d + 1 kernel with zero taps in between: the same sums
            w = torch.zeros((c, 1, (k - 1) * d + 1, (k - 1) * d + 1))
            w[:, 0, ::d, ::d] = torch.from_numpy(o['w']).reshape(c, k, k)
            y = F.conv2d(nchw(o, c), w, torch.from_numpy(o['b']), o['stride'], o['pad'], groups=c)
            acts[o['out']][..., o['out_off']:o['out_off'] + c] = q(act(y, o['relu']).permute(0, 2, 3, 1))
        elif kind == 'maxpool':
            y = F.max_pool2d(nchw(o, o['channels']), 3, o['stride'], 1)
            acts[o['out']][..., o['out_off']:o['out_off'] + o['channels']] = y.permute(0, 2, 3, 1)
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
