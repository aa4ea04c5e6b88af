"""Float64 references of the network ops of libpifpaf_b200 (include/pifpaf_b200.h), with the error bound a correct
kernel must meet.  Pure numpy; tests/test_kernel_refs.py checks them against torch in float64, tests/test_kernels_gpu.py
compares every kernel with them.  With `positions` (sample_positions) every reference is computed at chosen output
pixels only, reading just their receptive windows: tests/test_bench_shapes_gpu.py checks the benchmark's 64-image
forwards that way.

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


def gather(x, positions, iy, ix, fill=0.0):
    """x[b, iy, ix, :] in float64 for each row of positions (b = positions[:, 0]) -> [P, C]; `fill` where (iy, ix) lies
    outside x.  Only those pixels are read: x may be a view of a tensor of many GB."""
    H, W = x.shape[1:3]
    ok = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
    v = np.asarray(x[positions[:, 0], np.clip(iy, 0, H - 1), np.clip(ix, 0, W - 1)], dtype=np.float64)
    v[~ok] = fill
    return v


def conv_ref(x, w, b, stride, pad, groups=1, dilation=1, positions=None):
    """x [B, H, W, C] (NHWC), w [N, C / groups, k, k] (torch layout), b [N] or None, taps `dilation` pixels apart
    -> (y, mag): y = conv + b in float64 [B, Ho, Wo, N], mag = sum |x w| + |b| (the scale of the accumulation error).
    positions [P, 3] of output pixels (b, oy, ox): the same sums at those pixels only, [P, N]."""
    w = np.asarray(w, dtype=np.float64)
    C = x.shape[-1]
    N, cg, k, _ = w.shape
    assert C == cg * groups and N % groups == 0
    ng = N // groups
    if positions is None:
        x = np.asarray(x, dtype=np.float64)
        B, H, W, _ = x.shape
        Ho, Wo = out_hw(H, W, (k - 1) * dilation + 1, stride, pad)
        xp = np.zeros((B, H + 2 * pad, W + 2 * pad, C))
        xp[:, pad:pad + H, pad:pad + W] = x
        shape = (B, Ho, Wo, N)

        def window(y0, x0):
            return xp[:, y0:y0 + stride * (Ho - 1) + 1:stride, x0:x0 + stride * (Wo - 1) + 1:stride]
    else:
        iy0, ix0 = positions[:, 1] * stride - pad, positions[:, 2] * stride - pad
        shape = (len(positions), N)

        def window(y0, x0):
            return gather(x, positions, iy0 + y0, ix0 + x0)
    y = np.zeros(shape)
    mag = np.zeros(shape)
    for ky in range(k):
        for kx in range(k):
            xs = window(ky * dilation, kx * dilation)
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


def dw_gemm_ref(x, dw_w, dw_b, dw_relu, w, b, relu, positions=None):
    """fused depthwise 5x5 (stride 1, pad 2, f32 weights) -> 1x1 (bf16 weights) with a bf16 intermediate.
    x [B, H, W, C], dw_w [C, 5, 5], w [N, C] -> (ref, bound) of the bf16 output (at `positions` only, as conv_ref).
    The kernel rounds its f32 depthwise result d_gpu to bf16; |bf16(d_gpu) - d| <= 2^-8 |d| + (1 + 2^-8) e_dw, so the
    1x1 sees an operand error of at most that per k, weighted by |w_nk|."""
    C = x.shape[-1]
    d, dmag = conv_ref(x, np.asarray(dw_w).reshape(C, 1, 5, 5), dw_b, 1, 2, groups=C, positions=positions)
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


def heads_ref(a, w, b, n_fields, n_comp, comp_ops, upsample=1, positions=None):
    """CompositeField4 eval epilogue on a [B, h, w, K] feature map with weights w [N, K]: PixelShuffle(upsample) and the
    crop of (up - 1) // 2 low and ceil((up - 1) / 2) high cells, then the component ops with the index adds on the output
    grid -> per head (ref, bound) arrays [B, F, comp, h', w'] in float64.  The bound pushes the accumulation error through
    the activation (sigmoid: Lipschitz 1/4, softplus: 1) and adds a few f32 ulp for expf / log1pf / the index add.
    positions [P, 3] of output cells (b, oy, ox) on the h' x w' grid: the same values at those cells only, [P, F, comp]."""
    w = np.asarray(w, dtype=np.float64)
    up = upsample
    lo, hi = (up - 1) // 2, up // 2
    if positions is None:
        a = np.asarray(a, dtype=np.float64)
        B, h, wd, K = a.shape

        def fields(t, col, nf, nc):
            """conv channels (field, comp, sub-row, sub-column) -> [B, F, comp, h up, w up] (PixelShuffle), cropped"""
            t = t[..., col * up * up:(col + nf * nc) * up * up].reshape(B, h, wd, nf, nc, up, up)
            t = t.transpose(0, 3, 4, 1, 5, 2, 6).reshape(B, nf, nc, h * up, wd * up)
            return t[..., lo:h * up - hi, lo:wd * up - hi].copy()
    else:
        # output cell (oy, ox) is sub-pixel (sy, sx) of feature cell (cy, cx) before the crop
        (cy, sy), (cx, sx) = divmod(positions[:, 1] + lo, up), divmod(positions[:, 2] + lo, up)
        a = gather(a, positions, cy, cx)
        K = a.shape[-1]

        def fields(t, col, nf, nc):
            ch = col * up * up + (np.arange(nf * nc)[None, :] * up + sy[:, None]) * up + sx[:, None]
            return np.take_along_axis(t, ch, axis=1).reshape(-1, nf, nc)
    y = a @ w.T + b
    acc = (K + 2) * U_F32 * (np.abs(a) @ np.abs(w).T + np.abs(b))

    out, col, op_off = [], 0, 0
    for nf, nc in zip(n_fields, n_comp):
        v, e = fields(y, col, nf, nc), fields(acc, col, nf, nc)
        if positions is None:
            xs = np.arange(v.shape[-1], dtype=np.float64).reshape(1, 1, -1)
            ys = np.arange(v.shape[-2], dtype=np.float64).reshape(1, -1, 1)
        else:
            xs, ys = positions[:, 2:3].astype(np.float64), positions[:, 1:2].astype(np.float64)
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


def maxpool_ref(x, stride, positions=None):
    """3x3 max pool with padding 1 on x [B, H, W, C] (the values themselves: a max rounds nothing); at `positions`
    [P, 3] of output pixels only, as conv_ref"""
    if positions is not None:
        iy0, ix0 = positions[:, 1] * stride - 1, positions[:, 2] * stride - 1
        return np.max([gather(x, positions, iy0 + ky, ix0 + kx, -np.inf) for ky in range(3) for kx in range(3)], axis=0)
    B, H, W, C = x.shape
    Ho, Wo = out_hw(H, W, 3, stride, 1)
    xp = np.full((B, H + 2, W + 2, C), -np.inf, dtype=x.dtype)
    xp[:, 1:1 + H, 1:1 + W] = x
    return np.max([xp[:, ky:ky + stride * (Ho - 1) + 1:stride, kx:kx + stride * (Wo - 1) + 1:stride]
                   for ky in range(3) for kx in range(3)], axis=0)


def op_terms(o, taps, heads, images, batch, positions=None):
    """float64 reference of one op of network.build_ops on the tensors the GPU fed it -> (kind, [(got, ref, bound)]),
    one triple per output the op writes; bound None: compared exactly (the max pool).
    taps: tensor -> [>= batch, h, w, c_phys] after the forward, heads: the head outputs, images [B, 3, H, W] f32.
    positions [P, 3] of output pixels (b, oy, ox) (`sample_positions`): reference and bound at those pixels only, for
    every output channel, read from the receptive windows there; got, ref and bound are then [P, C] ([P, F, comp] for
    the heads)."""
    kind = o['kind']
    pos = positions

    def at(a):
        """a [B, h, w, ...] on the op's output grid -> its values at the positions (all of a without positions)"""
        return a if pos is None else a[pos[:, 0], pos[:, 1], pos[:, 2]]

    def a_in(t, off, n):
        return taps[t][:batch, ..., off:off + n]

    def out(n, t=None, off=None):
        t = o['out'] if t is None else t
        off = o.get('out_off', 0) if off is None else off
        return at(taps[t][:batch, ..., off:off + n])

    if kind == 'heads':
        refs = heads_ref(a_in(o['in'], 0, o['k_cols']), bf16_round(o['w']), o['b'], o['n_fields'], o['n_comp'],
                         o['ops'], o['upsample'], positions=pos)
        got = [hb[:batch] if pos is None else hb[pos[:, 0], :, :, pos[:, 1], pos[:, 2]] for hb in heads]
        return 'heads', [(g, r, bd) for g, (r, bd) in zip(got, refs)]
    if kind == 'input_conv':
        ref, mag = epilogue(*conv_ref(images[:batch].transpose(0, 2, 3, 1), o['w'], o['b'], o['stride'], o['pad'],
                                      positions=pos), o['relu'])
        return kind, [(out(o['c_out']), ref, bf16_bound(ref, mag, 3 * o['kernel'] ** 2))]
    if kind == 'maxpool':
        C = o['channels']
        return kind, [(out(C), maxpool_ref(a_in(o['in'], o['in_off'], C), o['stride'], positions=pos), None)]
    if kind == 'dw_conv1x1':
        C = o['channels']
        ref, bound = dw_gemm_ref(a_in(o['in'], o['in_off'], C), o['dw_w'], o['dw_b'], o['dw_relu'], bf16_round(o['w']),
                                 o['b'], o['relu'], positions=pos)
        return 'dw_gemm', [(out(cnt, t, col), ref[..., c0:c0 + cnt], bound[..., c0:c0 + cnt])
                           for c0, cnt, t, col in o['pieces']]
    if kind == 'dwconv':
        C, k, d = o['channels'], o['kernel'], o.get('dilation', 1)
        ref, mag = epilogue(*conv_ref(a_in(o['in'], o['in_off'], C), o['w'].reshape(C, 1, k, k), o['b'], o['stride'],
                                      o['pad'], groups=C, dilation=d, positions=pos), o['relu'])
        label = 'dwconv k%d s%d' % (k, o['stride']) + (' d%d' % d if d != 1 else '')
        return label, [(out(C), ref, bf16_bound(ref, mag, k * k))]
    if kind == 'conv':
        k, d = o['kernel'], o['dilation']
        ref, mag = conv_ref(a_in(o['in'], o['in_off'], o['c_in']), bf16_round(o['w']), o['b'], o['stride'], o['pad'],
                            dilation=d, positions=pos)
        res = None if o['residual'] < 0 else at(a_in(o['residual'], o['residual_off'], o['n_out']))
        ref, mag = epilogue(ref, mag, o['relu'], res)
        label = 'conv k%d' % k + (' d%d' % d if d != 1 else '')
        return label, [(out(o['n_out']), ref, bf16_bound(ref, mag, o['c_in'] * k * k))]
    assert kind == 'conv1x1', kind
    K, N = o['k_cols'], o['n_out']
    ref, mag = conv_ref(a_in(o['in'], o['in_off'], K), bf16_round(o['w'])[:, :, None, None], o['b'], 1, 0, positions=pos)
    ref, mag = epilogue(ref, mag, o['relu'])
    bound = bf16_bound(ref, mag, K)
    if 'pieces' in o:
        return 'gemm scatter', [(out(cnt, t, col), ref[..., c0:c0 + cnt], bound[..., c0:c0 + cnt])
                                for c0, cnt, t, col in o['pieces']]
    if o['shuffle_src'] >= 0:
        o_all = out(2 * N, off=0)
        assert np.array_equal(o_all[..., 0::2], at(a_in(o['shuffle_src'], o['shuffle_off'], N))), \
            'pass-through channels of the fused shuffle'
        return 'gemm shuffle', [(o_all[..., 1::2], ref, bound)]
    return 'gemm plain', [(out(N), ref, bound)]


def op_ref(o, taps, heads, images, batch, positions=None):
    """op_terms reduced to (kind, worst err / bound); the max pool is compared exactly (ratio 0 or inf)"""
    kind, terms = op_terms(o, taps, heads, images, batch, positions)
    return kind, max(worst_ratio(g, r, bd) if bd is not None else 0.0 if np.array_equal(g, r) else np.inf
                     for g, r, bd in terms)


TILE = (8, 16)              # output rows x columns of one CTA tile of the implicit-GEMM conv and depthwise kernels
GEMM_ROWS = 128             # rows (pixels) of one 1x1-GEMM tile over the flat [B h w] rows


BYTE_LIMITS = (2 ** 31, 2 ** 32)     # where a 32-bit byte offset, signed or not, wraps


def crossing_rows(n_pixels, c_phys, limits=BYTE_LIMITS, elem_bytes=2):
    """flat pixel rows of a [n_pixels, c_phys] tensor of elem_bytes-byte values whose bytes contain one of `limits`"""
    row = elem_bytes * c_phys
    return [x // row for x in limits if row and x < n_pixels * row]


def sample_positions(B, Ho, Wo, c_phys, seed, tile=TILE, n_random=4096, reads=(), limits=BYTE_LIMITS):
    """Output pixels (b, oy, ox) [P, 3] (sorted, unique) at which a B x Ho x Wo op is checked against op_terms: the
    union of
      - every pixel of rows {0, 1, Ho-2, Ho-1} and columns {0, 1, Wo-2, Wo-1} of images 0 and B-1 (padding, zero fill);
      - the four corners of every `tile` (rows x columns) output tile of image B-1;
      - GEMM tile edges on the flat M = B Ho Wo rows: rows m = 0 and 127 (mod 128) of the first and last three 128-row
        tiles, and row M-1;
      - for an output tensor (pitch c_phys, an int or one per tensor written) or an input tensor past 2^31 or 2^32
        bytes (`limits`), the output pixels within 2 rows of each crossing (crossing_rows).  reads: (H, W, c_phys, kernel,
        stride, pad, dilation) of each input tensor; an input crossing pixel selects every output whose window
        covers it;
      - n_random seeded uniform pixels of the whole batch."""
    M = B * Ho * Wo
    flat = []
    for b in sorted({0, B - 1}):
        for r in sorted({0, 1, Ho - 2, Ho - 1} & set(range(Ho))):
            flat.append((b * Ho + r) * Wo + np.arange(Wo))
        for c in sorted({0, 1, Wo - 2, Wo - 1} & set(range(Wo))):
            flat.append((b * Ho + np.arange(Ho)) * Wo + c)
    ty0, tx0 = np.arange(0, Ho, tile[0]), np.arange(0, Wo, tile[1])
    for ys in (ty0, np.minimum(ty0 + tile[0] - 1, Ho - 1)):
        for xs in (tx0, np.minimum(tx0 + tile[1] - 1, Wo - 1)):
            flat.append(((B - 1) * Ho + ys[:, None]) * Wo + xs[None, :])
    n_tiles = (M + GEMM_ROWS - 1) // GEMM_ROWS
    for t in sorted({0, 1, 2, n_tiles - 3, n_tiles - 2, n_tiles - 1} & set(range(n_tiles))):
        flat.append(np.minimum(t * GEMM_ROWS + np.array([0, GEMM_ROWS - 1]), M - 1))
    flat.append(np.array([M - 1]))
    for c in np.atleast_1d(c_phys):
        for m in crossing_rows(M, int(c), limits):
            flat.append(np.clip(np.arange(m - 2, m + 3), 0, M - 1))
    for (H, W, c, k, s, p, d) in reads:
        span = d * (k - 1) + 1
        for m in crossing_rows(B * H * W, c, limits):
            for mm in range(max(m - 2, 0), min(m + 3, B * H * W)):
                b, iy, ix = mm // (H * W), mm // W % H, mm % W
                oys = np.arange(max(-(-(iy + p - span + 1) // s), 0), min((iy + p) // s, Ho - 1) + 1)
                oxs = np.arange(max(-(-(ix + p - span + 1) // s), 0), min((ix + p) // s, Wo - 1) + 1)
                flat.append(((b * Ho + oys[:, None]) * Wo + oxs[None, :]).ravel())
    flat.append(np.random.default_rng(seed).integers(0, M, n_random))
    m = np.unique(np.concatenate([np.asarray(f, dtype=np.int64).ravel() for f in flat]))
    return np.stack([m // (Ho * Wo), m // Wo % Ho, m % Wo], axis=1)


def op_positions(o, tensors, B, seed, **kw):
    """sample_positions for op o of build_ops with tensors (h, w, c_phys) at batch B: its output grid, the pitches of
    the tensors it writes and the windows of the tensors it reads (kw: the other arguments of sample_positions)"""
    kind = o['kind']
    if kind == 'heads':
        h, w, _ = tensors[o['in']]
        up = o['upsample']
        return sample_positions(B, h * up - (up - 1), w * up - (up - 1), 0, seed, **kw)
    outs = [pc[2] for pc in o['pieces']] if 'pieces' in o else [o['out']]
    Ho, Wo, _ = tensors[outs[0]]
    if kind == 'input_conv':
        return sample_positions(B, Ho, Wo, [tensors[t][2] for t in outs], seed, **kw)
    if kind in ('conv', 'dwconv'):
        win = (o['kernel'], o['stride'], o['pad'], o.get('dilation', 1))
    elif kind == 'maxpool':
        win = (3, o['stride'], 1, 1)
    elif kind == 'dw_conv1x1':
        win = (o['kernel'], o['stride'], o['pad'], 1)
    else:
        win = (1, 1, 0, 1)
    reads = [(*tensors[o['in']], *win)]
    for t in (o.get('residual', -1), o.get('shuffle_src', -1)):
        if t >= 0:
            reads.append((*tensors[t], 1, 1, 0, 1))
    return sample_positions(B, Ho, Wo, [tensors[t][2] for t in outs], seed, reads=reads, **kw)


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
