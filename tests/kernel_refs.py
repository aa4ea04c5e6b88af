"""Float64 references of the network ops of libpifpaf_b200 (include/pifpaf_b200.h), with the error bound a correct
kernel must meet.  Pure numpy; tests/test_kernel_refs.py checks them against torch in float64, tests/test_kernels_gpu.py
compares every kernel with them.

Bound of one bf16 output (f32 accumulation of K products, then round to nearest even):
    |got - ref| <= 2^-8 |ref| + (K + 2) 2^-23 (sum |a w| + |b| + |res|)
the first term is the output rounding (half a bf16 ulp), the second the f32 accumulation (tensor-core adds may
truncate: a full f32 ulp per add).  Outputs kept in f32 (the heads) have no rounding term."""
import numpy as np

U_BF16 = 2.0 ** -8          # unit roundoff of bf16 (8-bit significand)
U_F32 = 2.0 ** -23          # one f32 ulp (relative)
SENTINEL = -12288.0         # exact in bf16 (-1.5 * 2^13); no op of the tests produces it
OP_RAW, OP_SIGMOID, OP_ADD_X, OP_ADD_Y, OP_SOFTPLUS = 0, 1, 2, 3, 4


def bf16_round(a):
    """float -> nearest bf16 value (ties to even), as float32."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    u = ((u + 0x7fff + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def bf16_truncate(a):
    """float -> bf16 by dropping the low 16 bits (rounding toward zero); only to show what the bound rejects."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    return (a.view(np.uint32) & np.uint32(0xffff0000)).view(np.float32)


def random_bf16(rng, shape, scale=1.0):
    return bf16_round(rng.standard_normal(shape) * scale)


def out_hw(h, w, kernel, stride, pad):
    return (h + 2 * pad - kernel) // stride + 1, (w + 2 * pad - kernel) // stride + 1


def conv_ref(x, w, b, stride, pad, groups=1, dilation=1):
    """x [B, H, W, C] (NHWC), w [N, C / groups, k, k] (torch layout), b [N] or None, taps `dilation` pixels apart
    -> (y, mag): y = conv + b in float64 [B, Ho, Wo, N], mag = sum |x w| + |b| (the scale of the accumulation error)."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    B, H, W, C = x.shape
    N, cg, k, _ = w.shape
    assert C == cg * groups and N % groups == 0
    ng = N // groups
    Ho, Wo = out_hw(H, W, (k - 1) * dilation + 1, stride, pad)
    xp = np.zeros((B, H + 2 * pad, W + 2 * pad, C))
    xp[:, pad:pad + H, pad:pad + W] = x
    y = np.zeros((B, Ho, Wo, N))
    mag = np.zeros((B, Ho, Wo, N))
    for ky in range(k):
        for kx in range(k):
            y0, x0 = ky * dilation, kx * dilation
            xs = xp[:, y0:y0 + stride * (Ho - 1) + 1:stride, x0:x0 + stride * (Wo - 1) + 1:stride]
            if groups == C and ng == 1:                  # depthwise: elementwise per channel
                y += xs * w[:, 0, ky, kx]
                mag += np.abs(xs) * np.abs(w[:, 0, ky, kx])
                continue
            for g in range(groups):
                xg = xs[..., g * cg:(g + 1) * cg]
                wg = w[g * ng:(g + 1) * ng, :, ky, kx]
                y[..., g * ng:(g + 1) * ng] += xg @ wg.T
                mag[..., g * ng:(g + 1) * ng] += np.abs(xg) @ np.abs(wg).T
    if b is not None:
        b = np.asarray(b, dtype=np.float64)
        y += b
        mag += np.abs(b)
    return y, mag


def bf16_bound(ref, mag, k_terms):
    """error bound of a bf16 output: ref and mag from conv_ref (mag including |b| and |res|)"""
    return U_BF16 * np.abs(ref) + (k_terms + 2) * U_F32 * mag


def epilogue(y, mag, code, res=None):
    """+ residual, then the activation of code (0 none, 1 ReLU, 2 ReLU6; the order of the torchvision block tail); both
    activations are 1-Lipschitz, the bound carries over"""
    assert code in (0, 1, 2), code
    if res is not None:
        res = np.asarray(res, dtype=np.float64)
        y = y + res
        mag = mag + np.abs(res)
    if code >= 1:
        y = np.maximum(y, 0.0)
    if code == 2:
        y = np.minimum(y, 6.0)
    return y, mag


def dw_gemm_ref(x, dw_w, dw_b, dw_relu, w, b, relu):
    """fused depthwise 5x5 (stride 1, pad 2, f32 weights) -> 1x1 (bf16 weights) with a bf16 intermediate.
    x [B, H, W, C], dw_w [C, 5, 5], w [N, C] -> (ref, bound) of the bf16 output.
    The kernel rounds its f32 depthwise result d_gpu to bf16; |bf16(d_gpu) - d| <= 2^-8 |d| + (1 + 2^-8) e_dw, so the
    1x1 sees an operand error of at most that per k, weighted by |w_nk|."""
    C = x.shape[-1]
    d, dmag = conv_ref(x, np.asarray(dw_w).reshape(C, 1, 5, 5), dw_b, 1, 2, groups=C)
    d, dmag = epilogue(d, dmag, dw_relu)
    e_dw = 27 * U_F32 * dmag
    d_err = U_BF16 * np.abs(d) + (1 + U_BF16) * e_dw
    w = np.asarray(w, dtype=np.float64)
    y = d @ w.T + np.asarray(b, dtype=np.float64)
    mag = np.abs(d) @ np.abs(w).T + np.abs(b)
    op_err = d_err @ np.abs(w).T
    y, mag = epilogue(y, mag, relu)
    return y, bf16_bound(y, mag, C) + op_err


def normalise_u8(images_hwc, mean, std):
    """torchvision ToTensor + Normalize in float32 with IEEE order: ((u / 255) - mean[c]) / std[c]; -> NHWC f32"""
    x = images_hwc.astype(np.float32) / np.float32(255.0)
    return (x - np.asarray(mean, dtype=np.float32)) / np.asarray(std, dtype=np.float32)


def heads_ref(a, w, b, n_fields, n_comp, comp_ops, upsample=1):
    """CompositeField4 eval epilogue on a [B, h, w, K] feature map with weights w [N, K]: PixelShuffle(upsample) and the
    crop of (up - 1) // 2 low and ceil((up - 1) / 2) high cells, then the component ops with the index adds on the output
    grid -> per head (ref, bound) arrays [B, F, comp, h', w'] in float64.  The bound pushes the accumulation error through
    the activation (sigmoid: Lipschitz 1/4, softplus: 1) and adds a few f32 ulp for expf / log1pf / the index add."""
    a = np.asarray(a, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    B, h, wd, K = a.shape
    up = upsample
    lo, hi = (up - 1) // 2, up // 2
    y = a @ w.T + b
    acc = (K + 2) * U_F32 * (np.abs(a) @ np.abs(w).T + np.abs(b))

    def fields(t, col, nf, nc):
        """conv channels (field, comp, sub-row, sub-column) -> [B, F, comp, h up, w up] (PixelShuffle), cropped"""
        t = t[..., col * up * up:(col + nf * nc) * up * up].reshape(B, h, wd, nf, nc, up, up)
        t = t.transpose(0, 3, 4, 1, 5, 2, 6).reshape(B, nf, nc, h * up, wd * up)
        return t[..., lo:h * up - hi, lo:wd * up - hi].copy()

    out, col, op_off = [], 0, 0
    for nf, nc in zip(n_fields, n_comp):
        v, e = fields(y, col, nf, nc), fields(acc, col, nf, nc)
        xs = np.arange(v.shape[-1], dtype=np.float64).reshape(1, 1, -1)
        ys = np.arange(v.shape[-2], dtype=np.float64).reshape(1, -1, 1)
        for c in range(nc):
            op = comp_ops[op_off + c]
            if op == OP_SIGMOID:
                v[:, :, c] = 1.0 / (1.0 + np.exp(-v[:, :, c]))
                e[:, :, c] = 0.25 * e[:, :, c] + 8 * 2.0 ** -24
            elif op == OP_ADD_X:
                v[:, :, c] += xs
                e[:, :, c] += 2.0 ** -24 * np.abs(v[:, :, c])
            elif op == OP_ADD_Y:
                v[:, :, c] += ys
                e[:, :, c] += 2.0 ** -24 * np.abs(v[:, :, c])
            elif op == OP_SOFTPLUS:
                v[:, :, c] = np.logaddexp(0.0, v[:, :, c])
                e[:, :, c] += 8 * 2.0 ** -24 * (np.abs(v[:, :, c]) + 1.0)
            else:
                e[:, :, c] += 2.0 ** -24 * np.abs(v[:, :, c])
        out.append((v, e))
        col += nf * nc
        op_off += nc
    return out


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound (> 1: the kernel is outside its error bound); NaN / inf in got count as infinite"""
    got = np.asarray(got, dtype=np.float64)
    err = np.abs(got - ref)
    err[~np.isfinite(got)] = np.inf
    return float((err / np.maximum(bound, 1e-300)).max()) if err.size else 0.0


def maxpool_ref(x, stride):
    """3x3 max pool with padding 1 on x [B, H, W, C] (the values themselves: a max rounds nothing)"""
    B, H, W, C = x.shape
    Ho, Wo = out_hw(H, W, 3, stride, 1)
    xp = np.full((B, H + 2, W + 2, C), -np.inf, dtype=x.dtype)
    xp[:, 1:1 + H, 1:1 + W] = x
    return np.max([xp[:, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride]
                   for ky in range(3) for kx in range(3)], axis=0)


def op_ref(o, taps, heads, images, batch):
    """float64 reference of one op of network.build_ops on the tensors the GPU fed it -> (kind, worst err / bound).
    taps: tensor -> [>= batch, h, w, c_phys] after the forward, heads: the head outputs, images [B, 3, H, W] f32.
    The max pool is compared exactly (ratio 0 or inf)."""
    kind = o['kind']

    def a_in(t, off, n):
        return taps[t][:batch, ..., off:off + n]

    def out(n, t=None, off=None):
        t = o['out'] if t is None else t
        off = o.get('out_off', 0) if off is None else off
        return taps[t][:batch, ..., off:off + n]

    if kind == 'heads':
        refs = heads_ref(a_in(o['in'], 0, o['k_cols']), bf16_round(o['w']), o['b'], o['n_fields'], o['n_comp'],
                         o['ops'], o['upsample'])
        return 'heads', max(worst_ratio(hb[:batch], r, bd) for hb, (r, bd) in zip(heads, refs))
    if kind == 'input_conv':
        ref, mag = epilogue(*conv_ref(images[:batch].transpose(0, 2, 3, 1), o['w'], o['b'], o['stride'], o['pad']),
                            o['relu'])
        return kind, worst_ratio(out(o['c_out']), ref, bf16_bound(ref, mag, 3 * o['kernel'] ** 2))
    if kind == 'maxpool':
        C = o['channels']
        return kind, 0.0 if np.array_equal(out(C), maxpool_ref(a_in(o['in'], o['in_off'], C), o['stride'])) else np.inf
    if kind == 'dw_conv1x1':
        C = o['channels']
        ref, bound = dw_gemm_ref(a_in(o['in'], o['in_off'], C), o['dw_w'], o['dw_b'], o['dw_relu'], bf16_round(o['w']),
                                 o['b'], o['relu'])
        return 'dw_gemm', max(worst_ratio(out(cnt, t, col), ref[..., c0:c0 + cnt], bound[..., c0:c0 + cnt])
                              for c0, cnt, t, col in o['pieces'])
    if kind == 'dwconv':
        C, k, d = o['channels'], o['kernel'], o.get('dilation', 1)
        ref, mag = epilogue(*conv_ref(a_in(o['in'], o['in_off'], C), o['w'].reshape(C, 1, k, k), o['b'], o['stride'],
                                      o['pad'], groups=C, dilation=d), o['relu'])
        label = 'dwconv k%d s%d' % (k, o['stride']) + (' d%d' % d if d != 1 else '')
        return label, worst_ratio(out(C), ref, bf16_bound(ref, mag, k * k))
    if kind == 'conv':
        k, d = o['kernel'], o['dilation']
        ref, mag = conv_ref(a_in(o['in'], o['in_off'], o['c_in']), bf16_round(o['w']), o['b'], o['stride'], o['pad'],
                            dilation=d)
        res = None if o['residual'] < 0 else a_in(o['residual'], o['residual_off'], o['n_out'])
        ref, mag = epilogue(ref, mag, o['relu'], res)
        label = 'conv k%d' % k + (' d%d' % d if d != 1 else '')
        return label, worst_ratio(out(o['n_out']), ref, bf16_bound(ref, mag, o['c_in'] * k * k))
    assert kind == 'conv1x1', kind
    K, N = o['k_cols'], o['n_out']
    ref, mag = conv_ref(a_in(o['in'], o['in_off'], K), bf16_round(o['w'])[:, :, None, None], o['b'], 1, 0)
    ref, mag = epilogue(ref, mag, o['relu'])
    bound = bf16_bound(ref, mag, K)
    if 'pieces' in o:
        return 'gemm scatter', max(worst_ratio(out(cnt, t, col), ref[..., c0:c0 + cnt], bound[..., c0:c0 + cnt])
                                   for c0, cnt, t, col in o['pieces'])
    if o['shuffle_src'] >= 0:
        o_all = out(2 * N, off=0)
        assert np.array_equal(o_all[..., 0::2], a_in(o['shuffle_src'], o['shuffle_off'], N)), \
            'pass-through channels of the fused shuffle'
        return 'gemm shuffle', worst_ratio(o_all[..., 1::2], ref, bound)
    return 'gemm plain', worst_ratio(out(N), ref, bound)


def written_columns(op, tensors):
    """(tensor, first column, end column) windows one op of network.build_ops writes ('heads' writes none of the
    activation tensors).  Plain outputs cover pad8(n) columns: the kernels store whole 8-channel vectors."""
    def pad8(v):
        return (v + 7) // 8 * 8
    kind = op['kind']
    if kind == 'input_conv':
        return [(op['out'], 0, pad8(op['c_out']))]
    if kind in ('conv1x1', 'dw_conv1x1') and 'pieces' in op:
        return [(t, col, col + cnt) for (_, cnt, t, col) in op['pieces']]
    if kind == 'conv1x1':
        if op['shuffle_src'] >= 0:
            return [(op['out'], 0, 2 * op['n_out'])]
        return [(op['out'], op['out_off'], op['out_off'] + pad8(op['n_out']))]
    if kind == 'conv':
        return [(op['out'], op['out_off'], op['out_off'] + pad8(op['n_out']))]
    if kind == 'dwconv':
        return [(op['out'], op['out_off'], op['out_off'] + pad8(op['channels']))]
    if kind == 'heads':
        return []
    raise ValueError(kind)
