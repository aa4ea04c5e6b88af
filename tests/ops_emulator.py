"""CPU (torch fp32) interpreter of the op list emitted by openpifpaf_b200.network.build_ops.

Test infrastructure: validates the host-side lowering (BN folding, physical channel
placement, fused cat+channel_shuffle, head epilogue ops) without a GPU by executing the
ops exactly as the C ABI documents them (include/pifpaf_b200.h) and comparing with the
oracle network."""
import numpy as np
import torch
import torch.nn.functional as F


def run_ops(tensors, ops, images, bf16=False):
    """images [B,3,H,W] float32 -> list of head outputs [B,F,comp,h,w].

    With ``bf16`` activations and the weights of the GEMM-like ops (1x1, implicit-GEMM conv, heads) are rounded to bf16;
    depthwise and stem weights stay f32, as the kernels read them."""
    B = images.shape[0]
    acts = [torch.zeros((B, h, w, c), dtype=torch.float32) for (h, w, c) in tensors]

    def q(x):
        return x.to(torch.bfloat16).to(torch.float32) if bf16 else x

    heads_out = None
    for o in ops:
        kind = o['kind']
        if kind == 'input_conv':
            y = F.conv2d(images, torch.from_numpy(o['w']), torch.from_numpy(o['b']), o['stride'], o['pad'])
            if o['relu']:
                y = F.relu(y)
            acts[o['out']][..., :o['c_out']] = q(y.permute(0, 2, 3, 1))
        elif kind == 'conv1x1':
            a = acts[o['in']][..., o['in_off']:o['in_off'] + o['k_cols']]
            w, b = q(torch.from_numpy(o['w'])), torch.from_numpy(o['b'])
            y = a @ w.t() + b
            if o['relu']:
                y = F.relu(y)
            y = q(y)
            n = o['n_out']
            out = acts[o['out']]
            if 'pieces' in o:
                for (c0, cnt, t_id, t_col) in o['pieces']:
                    acts[t_id][..., t_col:t_col + cnt] = y[..., c0:c0 + cnt]
            elif o['shuffle_src'] < 0:
                out[..., o['out_off']:o['out_off'] + n] = y
            else:
                src = acts[o['shuffle_src']][..., o['shuffle_off']:o['shuffle_off'] + n]
                out[..., 0:2 * n:2] = src
                out[..., 1:2 * n:2] = y
        elif kind == 'conv':
            a = acts[o['in']][..., o['in_off']:o['in_off'] + o['c_in']].permute(0, 3, 1, 2)
            y = F.conv2d(a, q(torch.from_numpy(o['w'])), torch.from_numpy(o['b']), o['stride'], o['pad'])
            y = y.permute(0, 2, 3, 1)
            if o['residual'] >= 0:
                y = y + acts[o['residual']][..., o['residual_off']:o['residual_off'] + o['n_out']]
            if o['relu']:
                y = F.relu(y)
            acts[o['out']][..., o['out_off']:o['out_off'] + o['n_out']] = q(y)
        elif kind == 'dw_conv1x1':
            c = o['channels']
            a = acts[o['in']][..., o['in_off']:o['in_off'] + c].permute(0, 3, 1, 2)
            wdw = torch.from_numpy(o['dw_w']).reshape(c, 1, o['kernel'], o['kernel'])
            y = F.conv2d(a, wdw, torch.from_numpy(o['dw_b']), o['stride'], o['pad'], groups=c)
            if o['dw_relu']:
                y = F.relu(y)
            y = q(y.permute(0, 2, 3, 1))                    # the bf16 A operand of the fused GEMM
            y = y @ q(torch.from_numpy(o['w'])).t() + torch.from_numpy(o['b'])
            if o['relu']:
                y = F.relu(y)
            y = q(y)
            for (c0, cnt, t_id, t_col) in o['pieces']:
                acts[t_id][..., t_col:t_col + cnt] = y[..., c0:c0 + cnt]
        elif kind == 'dwconv':
            c = o['channels']
            a = acts[o['in']][..., o['in_off']:o['in_off'] + c].permute(0, 3, 1, 2)
            w = torch.from_numpy(o['w']).reshape(c, 1, o['kernel'], o['kernel'])
            y = F.conv2d(a, w, torch.from_numpy(o['b']), o['stride'], o['pad'], groups=c)
            if o['relu']:
                y = F.relu(y)
            acts[o['out']][..., o['out_off']:o['out_off'] + c] = q(y.permute(0, 2, 3, 1))
        elif kind == 'heads':
            a = acts[o['in']][..., :o['k_cols']]
            y = a @ q(torch.from_numpy(o['w'])).t() + torch.from_numpy(o['b'])   # [B,h,w,N]
            _, h, w, _ = y.shape
            xs = torch.arange(w, dtype=torch.float32).view(1, 1, w)
            ys = torch.arange(h, dtype=torch.float32).view(1, h, 1)
            heads_out, col, op_off = [], 0, 0
            for nf, nc in zip(o['n_fields'], o['n_comp']):
                t = y[..., col:col + nf * nc].reshape(B, h, w, nf, nc).permute(0, 3, 4, 1, 2).clone()
                for c_i in range(nc):
                    op = o['ops'][op_off + c_i]
                    if op == 1:
                        t[:, :, c_i] = torch.sigmoid(t[:, :, c_i])
                    elif op == 2:
                        t[:, :, c_i] += xs
                    elif op == 3:
                        t[:, :, c_i] += ys
                    elif op == 4:
                        t[:, :, c_i] = F.softplus(t[:, :, c_i])
                heads_out.append(t)
                col += nf * nc
                op_off += nc
        else:
            raise ValueError(kind)
    return heads_out, acts
