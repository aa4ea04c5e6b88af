"""CPU: the float64 references of tests/kernel_refs.py against torch in float64, the bound they come with, and the
write-once property of the op lists that the teacher-forced checks of tests/test_kernels_gpu.py rely on."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_refs as kr
from openpifpaf_b200 import network
from oracle import net_oracle


def torch_conv(x_nhwc, w, b, stride, pad, groups=1, dilation=1):
    x = torch.from_numpy(np.asarray(x_nhwc, dtype=np.float64)).permute(0, 3, 1, 2)
    y = F.conv2d(x, torch.from_numpy(np.asarray(w, dtype=np.float64)),
                 None if b is None else torch.from_numpy(np.asarray(b, dtype=np.float64)), stride, pad, dilation, groups)
    return y.permute(0, 2, 3, 1).numpy()


@pytest.mark.parametrize('k,stride,pad,c_in,n_out,groups', [
    (1, 1, 0, 24, 40, 1),       # pointwise
    (1, 2, 0, 16, 8, 1),        # strided 1x1 (ResNet downsample)
    (3, 1, 1, 7, 5, 1),         # dense
    (3, 2, 0, 6, 4, 1),         # strided, no padding
    (7, 2, 3, 3, 16, 1),        # stem
    (5, 1, 2, 12, 12, 12),      # depthwise
    (5, 2, 1, 9, 9, 9),         # depthwise, stride 2
    (3, 1, 1, 8, 12, 4),        # grouped
])
def test_conv_ref_matches_torch_float64(k, stride, pad, c_in, n_out, groups):
    rng = np.random.default_rng(k * 100 + c_in)
    x = rng.standard_normal((2, 11, 9, c_in))
    w = rng.standard_normal((n_out, c_in // groups, k, k))
    b = rng.standard_normal(n_out)
    y, mag = kr.conv_ref(x, w, b, stride, pad, groups=groups)
    want = torch_conv(x, w, b, stride, pad, groups)
    assert y.shape == want.shape
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-12)
    # mag is the same conv on absolute values
    np.testing.assert_allclose(mag, torch_conv(np.abs(x), np.abs(w), np.abs(b), stride, pad, groups), rtol=1e-12)


@pytest.mark.parametrize('k,stride,pad,dilation,c_in,n_out,groups', [
    (3, 1, 2, 2, 8, 6, 1),      # ResNet block 5 under --resnet-block5-dilation 2
    (3, 1, 4, 4, 5, 7, 1),      # dilation 4: most taps in the padding
    (3, 1, 0, 2, 6, 4, 1),      # no padding: the output shrinks by d (k - 1)
    (5, 1, 4, 2, 12, 12, 12),   # depthwise 5x5, dilation 2 (--shufflenetv2k-stage4-dilation 2)
    (5, 1, 6, 3, 9, 9, 9),      # depthwise, dilation 3
    (3, 2, 2, 2, 4, 4, 4),      # strided (the kernels refuse it; the reference is still a conv)
])
def test_conv_ref_dilated_matches_torch_float64(k, stride, pad, dilation, c_in, n_out, groups):
    rng = np.random.default_rng(k * 100 + c_in + dilation)
    x = rng.standard_normal((2, 13, 11, c_in))
    w = rng.standard_normal((n_out, c_in // groups, k, k))
    b = rng.standard_normal(n_out)
    y, mag = kr.conv_ref(x, w, b, stride, pad, groups=groups, dilation=dilation)
    want = torch_conv(x, w, b, stride, pad, groups, dilation)
    assert y.shape == want.shape
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(mag, torch_conv(np.abs(x), np.abs(w), np.abs(b), stride, pad, groups, dilation), rtol=1e-12)


@pytest.mark.parametrize('code', [0, 1, 2])
def test_epilogue_activation_codes(code):
    """codes 0 / 1 / 2 of include/pifpaf_b200.h (none, ReLU, ReLU6) after the residual add"""
    rng = np.random.default_rng(7)
    y = rng.uniform(-4.0, 10.0, (2, 5, 6, 8))
    res = rng.standard_normal((2, 5, 6, 8))
    mag = np.abs(y)
    got, got_mag = kr.epilogue(y, mag, code, res)
    t = torch.from_numpy(y + res)
    want = [t, F.relu(t), F.relu6(t)][code].numpy()
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got_mag, mag + np.abs(res))
    if code == 2:
        assert (got == 6).any() and (got == 0).any()


def test_maxpool_ref_matches_torch():
    rng = np.random.default_rng(8)
    for stride in (1, 2):
        for H, W in ((1, 1), (2, 3), (9, 8), (10, 7)):
            x = rng.standard_normal((2, H, W, 5))
            want = F.max_pool2d(torch.from_numpy(x).permute(0, 3, 1, 2), 3, stride, 1).permute(0, 2, 3, 1).numpy()
            np.testing.assert_array_equal(kr.maxpool_ref(x, stride), want)


def test_residual_epilogue_adds_before_relu():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((1, 6, 5, 8))
    w = rng.standard_normal((8, 8, 3, 3))
    b = rng.standard_normal(8)
    res = rng.standard_normal((1, 6, 5, 8))
    y, mag = kr.conv_ref(x, w, b, 1, 1)
    y, mag = kr.epilogue(y, mag, True, res)
    want = np.maximum(torch_conv(x, w, b, 1, 1) + res, 0.0)
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-12)
    assert (mag >= np.abs(res)).all()


def test_dw_gemm_ref_is_depthwise_then_pointwise():
    rng = np.random.default_rng(2)
    C, N = 10, 6
    x = rng.standard_normal((2, 7, 9, C))
    dw_w = rng.standard_normal((C, 5, 5))
    dw_b = rng.standard_normal(C)
    w = rng.standard_normal((N, C))
    b = rng.standard_normal(N)
    y, bound = kr.dw_gemm_ref(x, dw_w, dw_b, 1, w, b, 1)
    d = np.maximum(torch_conv(x, dw_w.reshape(C, 1, 5, 5), dw_b, 1, 2, groups=C), 0.0)
    want = np.maximum(torch_conv(d, w.reshape(N, C, 1, 1), b, 1, 0), 0.0)
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-12)
    # the bf16 intermediate term dominates the bound: at least 2^-8 sum_k |w_nk| |d_k|
    assert (bound >= kr.U_BF16 * (np.abs(d) @ np.abs(w).T) - 1e-12).all()


def torch_heads(a, wt, bias, n_fields, n_comp, comp_ops, up):
    """the heads epilogue in torch float64: conv as a matmul, PixelShuffle(up), the reference's crop, the component ops"""
    B = a.shape[0]
    y = (torch.from_numpy(a) @ torch.from_numpy(wt).T + torch.from_numpy(bias)).permute(0, 3, 1, 2)
    out, col, off = [], 0, 0
    for nf, nc in zip(n_fields, n_comp):
        t = torch.nn.PixelShuffle(up)(y[:, col * up * up:(col + nf * nc) * up * up])
        lo, hi = (up - 1) // 2, int(np.ceil((up - 1) / 2.0))
        t = t[:, :, lo:t.shape[2] - hi, lo:t.shape[3] - hi]
        h, w = t.shape[2:]
        t = t.reshape(B, nf, nc, h, w).clone()
        for c in range(nc):
            op = comp_ops[off + c]
            if op == 1:
                t[:, :, c] = torch.sigmoid(t[:, :, c])
            elif op == 2:
                t[:, :, c] += torch.arange(w, dtype=torch.float64).view(1, 1, w)
            elif op == 3:
                t[:, :, c] += torch.arange(h, dtype=torch.float64).view(1, h, 1)
            elif op == 4:
                t[:, :, c] = F.softplus(t[:, :, c])
        out.append(t.numpy())
        col += nf * nc
        off += nc
    return out


def check_heads_ref(up):
    rng = np.random.default_rng(3)
    B, h, w, K = 2, 5, 7, 24
    n_fields, n_comp = [3, 2], [5, 9]
    comp_ops = [1, 2, 3, 4, 0] + [1, 2, 3, 0, 0, 4, 4, 1, 0]
    N = sum(f * c for f, c in zip(n_fields, n_comp)) * up * up
    a = rng.standard_normal((B, h, w, K))
    wt = rng.standard_normal((N, K)) * 3
    bias = rng.standard_normal(N)
    got = kr.heads_ref(a, wt, bias, n_fields, n_comp, comp_ops, up)
    for (v, e), want in zip(got, torch_heads(a, wt, bias, n_fields, n_comp, comp_ops, up)):
        assert v.shape == want.shape == (B, v.shape[1], v.shape[2], h * up - (up - 1), w * up - (up - 1))
        # torch's softplus returns x above 20 (threshold): log1p(exp(-20)) = 2e-9 from the exact value
        np.testing.assert_allclose(v, want, rtol=1e-12, atol=3e-9)
        assert (e > 0).all()


def test_heads_ref_matches_torch_ops():
    check_heads_ref(1)


@pytest.mark.parametrize('up', [2, 3])
def test_heads_ref_upsampled_matches_torch_ops(up):
    """upsample_stride > 1 (heads.py:307-343): PixelShuffle, the crop, and the index adds on the output grid"""
    check_heads_ref(up)


def test_bf16_round_is_torch_round_to_nearest_even():
    rng = np.random.default_rng(4)
    a = np.concatenate([rng.standard_normal(100000).astype(np.float32) * 1e3,
                        np.array([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 2 ** -130], dtype=np.float32)])
    want = torch.from_numpy(a).to(torch.bfloat16).to(torch.float32).numpy()
    np.testing.assert_array_equal(kr.bf16_round(a), want)
    assert kr.bf16_round(np.float32(kr.SENTINEL)) == np.float32(kr.SENTINEL)


def test_bound_accepts_round_to_nearest_and_rejects_truncation():
    """the bf16 bound is tight enough to see half an ulp: f32 results rounded to nearest pass, truncated ones fail"""
    rng = np.random.default_rng(5)
    x = kr.random_bf16(rng, (2, 9, 9, 64))
    w = kr.random_bf16(rng, (48, 64, 1, 1), 1 / 8)
    ref, mag = kr.conv_ref(x, w, None, 1, 0)
    f32 = ref.astype(np.float32)
    bound = kr.bf16_bound(ref, mag, 64)
    assert kr.worst_ratio(kr.bf16_round(f32), ref, bound) <= 1.0
    assert kr.worst_ratio(kr.bf16_truncate(f32), ref, bound) > 1.0
    assert kr.worst_ratio(np.where(ref > 0, np.nan, f32), ref, bound) == np.inf


def test_normalise_u8_is_torchvision_order():
    rng = np.random.default_rng(6)
    u = rng.integers(0, 256, (2, 5, 7, 3), dtype=np.uint8)
    mean, std = network.CompiledNet.IMAGE_MEAN, network.CompiledNet.IMAGE_STD
    t = torch.from_numpy(u).to(torch.float32) / 255.0
    want = (t - torch.tensor(mean, dtype=torch.float32)) / torch.tensor(std, dtype=torch.float32)
    np.testing.assert_array_equal(kr.normalise_u8(u, mean, std), want.numpy())


def _write_once(tensors, ops):
    owner = [np.full(c, -1) for (_, _, c) in tensors]
    for i, o in enumerate(ops):
        for t, c0, c1 in kr.written_columns(o, tensors):
            assert 0 <= c0 < c1 <= tensors[t][2], (i, o['kind'], t, c0, c1)
            clash = owner[t][c0:c1]
            assert (clash < 0).all(), f'op {i} ({o["kind"]}) writes tensor {t} columns owned by op {clash.max()}'
            owner[t][c0:c1] = i
    return owner


@pytest.mark.parametrize('base,layout,fuse', [
    ('shufflenetv2k16', 'bins', True), ('shufflenetv2k16', 'bins', False), ('shufflenetv2k16', 'shuffle', False),
    ('shufflenetv2k30', 'bins', False), ('resnet18', None, None), ('resnet50', None, None)])
def test_every_tensor_column_is_written_by_one_op(base, layout, fuse):
    """each (tensor, column) is written by at most one op of a forward: a tap after the forward shows every op's
    output as that op left it, and every op's inputs as it read them"""
    if base.startswith('resnet'):
        plan = network.plan_from_shell(net_oracle.make_shell(base, seed=0))
        tensors, ops, _ = network.build_ops(plan, 97, 129)
    else:
        plan = network.random_plan(base, seed=0)
        tensors, ops, _ = network.build_ops(plan, 97, 129, layout=layout, fuse_dw=fuse)
    owner = _write_once(tensors, ops)
    # and every column an op reads was produced before it (or is never written: zero padding)
    for i, o in enumerate(ops):
        if o['kind'] == 'input_conv':
            continue
        width = o.get('k_cols', o.get('channels', o.get('c_in')))
        reads = [(o['in'], o.get('in_off', 0), width)]
        if o.get('shuffle_src', -1) >= 0:
            reads.append((o['shuffle_src'], o['shuffle_off'], o['n_out']))
        if o.get('residual', -1) >= 0:
            reads.append((o['residual'], o['residual_off'], o['n_out']))
        for t, c0, n in reads:
            assert (owner[t][c0:c0 + n] < i).all(), (i, o['kind'], t)


def _emulation_plan(name):
    import det_models
    import mobilenetv2_models as mm
    import shufflenetv2k_models as sm
    if name == 'mobilenetv2':
        return network.plan_from_shell(mm.make_pose_shell(seed=0))
    if name in det_models.VARIANTS:
        return network.plan_from_shell(det_models.make_variant_shell(name, seed=0))
    return network.plan_from_shell(sm.make_pose_shell(name, 'tiny', seed=0))


@pytest.mark.parametrize('name,layout,fuse', [
    ('dil2_conv5stage', 'bins', True), ('conv2_dil2', 'shuffle', False), ('cocodet', None, None), ('pool2', None, None),
    ('dil4', None, None), ('mobilenetv2', None, None)])
def test_op_ref_bounds_hold_for_the_bf16_emulation(name, layout, fuse):
    """kernel_refs.op_ref on every op kind (dilated convs, max pool, upsampled heads, scatter, shuffle, fused depthwise
    -> 1x1): ops_emulator.run_ops with bf16 rounds where the kernels round, so its tensors must meet every bound"""
    import ops_emulator
    kw = {} if layout is None else {'layout': layout, 'fuse_dw': fuse}
    tensors, ops, _ = network.build_ops(_emulation_plan(name), 49, 65, **kw)
    images = np.random.default_rng(1).standard_normal((2, 3, 49, 65)).astype(np.float32)
    heads, acts = ops_emulator.run_ops(tensors, ops, torch.from_numpy(images), bf16=True)
    taps = {t: a.numpy() for t, a in enumerate(acts)}
    kinds = set()
    for i, o in enumerate(ops):
        kind, r = kr.op_ref(o, taps, [h.numpy() for h in heads], images, 2)
        assert r <= 1.0, (i, kind, r)
        kinds.add(kind)
    print(name, sorted(kinds))


def _emulated(name, layout=None, fuse=None, u8=False, H=49, W=65, B=2):
    """build_ops of an emulation plan and its bf16 emulation (ops_emulator.run_ops) on seeded images; u8: the images
    are raw uint8 ones normalised as the uint8 stem does (kernel_refs.normalise_u8)"""
    import ops_emulator
    kw = {} if layout is None else {'layout': layout, 'fuse_dw': fuse}
    tensors, ops, _ = network.build_ops(_emulation_plan(name), H, W, **kw)
    rng = np.random.default_rng(1)
    if u8:
        raw = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
        images = np.ascontiguousarray(
            kr.normalise_u8(raw, network.CompiledNet.IMAGE_MEAN, network.CompiledNet.IMAGE_STD).transpose(0, 3, 1, 2))
    else:
        images = rng.standard_normal((B, 3, H, W)).astype(np.float32)
    heads, acts = ops_emulator.run_ops(tensors, ops, torch.from_numpy(images), bf16=True)
    return tensors, ops, {t: a.numpy() for t, a in enumerate(acts)}, [h.numpy() for h in heads], images


def _at(a, pos, heads=False):
    """a full-size op_terms array at positions: [B, h, w, C] -> [P, C]; head outputs [B, F, comp, h, w] -> [P, F, comp]"""
    return a[pos[:, 0], :, :, pos[:, 1], pos[:, 2]] if heads else a[pos[:, 0], pos[:, 1], pos[:, 2]]


@pytest.mark.parametrize('name,layout,fuse,u8', [
    ('dil2_conv5stage', 'bins', True, False), ('conv2_dil2', 'shuffle', False, False), ('cocodet', None, None, False),
    ('pool2', None, None, True), ('dil4', None, None, False), ('mobilenetv2', None, None, True)])
def test_sampled_op_terms_equal_the_full_reference(name, layout, fuse, u8):
    """op_terms at sample_positions (every op kind, float and uint8-normalised stems) is the full reference, bound and
    output restricted to those positions"""
    tensors, ops, taps, heads, images = _emulated(name, layout, fuse, u8)
    kinds = set()
    for i, o in enumerate(ops):
        pos = kr.op_positions(o, tensors, 2, seed=i, n_random=64)
        kind, full = kr.op_terms(o, taps, heads, images, 2)
        kind_s, sampled = kr.op_terms(o, taps, heads, images, 2, positions=pos)
        assert kind_s == kind and len(sampled) == len(full)
        for (g, r, bd), (gs, rs, bds) in zip(full, sampled):
            assert np.array_equal(_at(g, pos, kind == 'heads'), gs), (i, kind)
            np.testing.assert_allclose(rs, _at(r, pos, kind == 'heads'), rtol=1e-12, atol=1e-12, err_msg=f'{i} {kind}')
            if bd is None:
                assert bds is None
            else:
                np.testing.assert_allclose(bds, _at(bd, pos, kind == 'heads'), rtol=1e-12, atol=1e-15)
        assert kr.op_ref(o, taps, heads, images, 2, positions=pos)[1] <= 1.0, (i, kind)
        kinds.add(kind)
    print(name, sorted(kinds))


def test_sampled_op_kinds_cover_every_kind():
    """the plans above reach every label op_terms gives: each sampled path was compared"""
    kinds = set()
    for name, layout, fuse in (('dil2_conv5stage', 'bins', True), ('conv2_dil2', 'shuffle', False),
                               ('cocodet', None, None), ('pool2', None, None), ('dil4', None, None),
                               ('mobilenetv2', None, None)):
        kw = {} if layout is None else {'layout': layout, 'fuse_dw': fuse}
        _, ops, _ = network.build_ops(_emulation_plan(name), 49, 65, **kw)
        for o in ops:
            kinds.add(o['kind'] + ('-pieces' if 'pieces' in o else '') + ('-shuffle' if o.get('shuffle_src', -1) >= 0 else '')
                      + ('-res' if o.get('residual', -1) >= 0 else '') + ('-dil' if o.get('dilation', 1) > 1 else '')
                      + ('-up' if o.get('upsample', 1) > 1 else ''))
    want = {'input_conv', 'conv', 'conv-res', 'conv-dil', 'conv1x1', 'conv1x1-pieces', 'conv1x1-shuffle', 'dwconv',
            'dwconv-dil', 'dw_conv1x1-pieces', 'maxpool', 'heads', 'heads-up'}
    assert want <= kinds, want - kinds


def _defect_case():
    """the emulated mobilenetv2 and its first plain implicit-GEMM conv with an output of at least 16 x 32 pixels"""
    tensors, ops, taps, heads, images = _emulated('mobilenetv2', H=65, W=129)
    i = next(i for i, o in enumerate(ops) if o['kind'] == 'conv' and tensors[o['out']][0] >= 16
             and tensors[o['out']][1] >= 32)
    return tensors, ops, taps, heads, images, i


@pytest.mark.parametrize('where', ['last pixel', 'tile corner', 'crossing row'])
def test_sampled_reference_reports_one_wrong_value(where):
    """a single wrong value in the emulated output of one op is reported (ratio > 1) by the sampled reference without
    any random positions: at the last pixel of the last image, at a corner of an 8 x 16 tile of the last image, and at
    the pixel row holding a (here synthetic) 32-bit offset crossing of the output"""
    tensors, ops, taps, heads, images, i = _defect_case()
    o = ops[i]
    B = 2
    Ho, Wo, c = tensors[o['out']]
    limits = kr.BYTE_LIMITS
    if where == 'last pixel':
        b, y, x = B - 1, Ho - 1, Wo - 1
    elif where == 'tile corner':
        b, y, x = B - 1, 2 * kr.TILE[0] - 1, kr.TILE[1]        # bottom-left corner of the second tile row's 2nd tile
    else:
        m = (B * Ho * Wo) * 3 // 5 + 7                           # an interior pixel no other class selects
        b, y, x = m // (Ho * Wo), m // Wo % Ho, m % Wo
        limits = (m * 2 * c + c,)                                # a byte limit inside that pixel row
    pos = kr.op_positions(o, tensors, B, seed=0, n_random=0, limits=limits)
    assert kr.op_ref(o, taps, heads, images, B, positions=pos)[1] <= 1.0
    if where == 'crossing row':
        clean = kr.op_positions(o, tensors, B, seed=0, n_random=0)
        assert not ((clean == (b, y, x)).all(1)).any(), 'the crossing row alone must select the pixel'
    bad = dict(taps)
    bad[o['out']] = taps[o['out']].copy()
    v = bad[o['out']][b, y, x, o['n_out'] // 2]
    bad[o['out']][b, y, x, o['n_out'] // 2] = v + 1.0 + 0.25 * abs(v)      # far outside the bound at any magnitude
    kind, r = kr.op_ref(o, bad, heads, images, B, positions=pos)
    assert r > 1.0, (where, kind, r)


def test_sample_positions_hold_every_class():
    """the benchmark's stage-2 entry: t_c (64 x 321 x 321 x 192 bf16 = 2 532 335 616 B) written by a 1x1 GEMM and read
    by the stride-2 depthwise 5x5; both ops' positions hold the pixels around byte 2^31 (row 5 592 405, image 54)"""
    import bench
    cfg = bench.CONFIGS['C0']
    tensors, ops, _ = network.build_ops(bench.make_plan(cfg), 641, 641)
    B = 64
    big = [t for t, (h, w, c) in enumerate(tensors) if B * h * w * c * 2 > 2 ** 31]
    assert len(big) == 1 and tensors[big[0]] == (321, 321, 192)
    assert kr.crossing_rows(B * 321 * 321, 192) == [5592405]
    writer = next(o for o in ops if o.get('out') == big[0] and o['kind'] == 'conv1x1')
    reader = next(o for o in ops if o.get('in') == big[0])
    assert reader['kind'] == 'dwconv' and reader['stride'] == 2 and reader['kernel'] == 5
    pw = kr.op_positions(writer, tensors, B, seed=1)
    dw = kr.op_positions(reader, tensors, B, seed=2)

    def has(pos, pts):
        s = {tuple(p) for p in pos.tolist()}
        return all(tuple(p) in s for p in pts)
    assert has(pw, [(m // 321 ** 2, m // 321 % 321, m % 321) for m in range(5592403, 5592408)])
    assert (54, 87, 264) == (5592405 // 321 ** 2, 5592405 // 321 % 321, 5592405 % 321)
    # outputs oy 43..44 / ox 131..133 of the stride-2 window (pad 2) cover input pixel (87, 264)
    assert has(dw, [(54, y, x) for y in (43, 44) for x in (131, 132, 133)])
    for pos, (Ho, Wo) in ((pw, (321, 321)), (dw, (161, 161))):
        M = B * Ho * Wo
        assert (pos[:, 0] < B).all() and (pos[:, 1] < Ho).all() and (pos[:, 2] < Wo).all()
        edge = [(b, r, x) for b in (0, B - 1) for r in (0, 1, Ho - 2, Ho - 1) for x in range(Wo)]
        edge += [(b, y, c) for b in (0, B - 1) for c in (0, 1, Wo - 2, Wo - 1) for y in range(Ho)]
        corners = [(B - 1, y, x) for y0 in range(0, Ho, 8) for x0 in range(0, Wo, 16)
                   for y in (y0, min(y0 + 7, Ho - 1)) for x in (x0, min(x0 + 15, Wo - 1))]
        n_t = (M + 127) // 128
        rows = [min(t * 128 + r, M - 1) for t in (0, 1, 2, n_t - 3, n_t - 2, n_t - 1) for r in (0, 127)] + [M - 1]
        assert has(pos, edge) and has(pos, corners)
        assert has(pos, [(m // (Ho * Wo), m // Wo % Ho, m % Wo) for m in rows])
        structured = len({*edge, *corners})
        assert structured + 3500 < len(pos) < structured + 4200, len(pos)      # ~4096 random ones besides
        print('positions', Ho, Wo, len(pos))
