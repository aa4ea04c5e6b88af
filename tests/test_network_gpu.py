"""GPU: backbone + heads kernels against the plain PyTorch fp32 reference of the same network, and the
end-to-end Predictor path (network fields -> CUDA decoder) against the oracle decoder on the same fields."""
import numpy as np
import pytest
import torch

import helpers
import ops_emulator
from openpifpaf_b200 import constants, network, predictor
from oracle import cifcaf as oc, net_oracle

pytestmark = pytest.mark.gpu

# bf16 activations / weights with f32 accumulation through ~57 fused ops, against fp32 PyTorch:
# tolerance relative to the standard deviation of each field tensor (stated per BASELINE north_star 'bf16')
FIELD_TOL_REL = 3e-2


@pytest.fixture(scope='module')
def small():
    shell = net_oracle.make_shell('shufflenetv2k16', seed=1)
    plan = network.plan_from_shell(shell)
    return shell, plan


@pytest.mark.parametrize('layout,fuse', [('bins', True), ('bins', False), ('shuffle', False)])
def test_every_op_matches_bf16_emulation(small, layout, fuse):
    """each fused op against a CPU emulation that rounds to bf16 at the same points (wgmma and SIMT debug),
    for both activation layouts (scatter GEMMs into per-block bins / fused cat+shuffle epilogue) and with the
    depthwise -> 1x1 pairs of the stride-1 blocks as one kernel (k_dw_gemm) or two."""
    shell, plan = small
    h, w, B = 97, 129, 2
    x = torch.randn(B, 3, h, w, generator=torch.Generator().manual_seed(0))
    tensors, ops, _ = network.build_ops(plan, h, w, layout=layout, fuse_dw=fuse)
    assert any(o['kind'] == 'dw_conv1x1' for o in ops) == fuse
    emu_heads, emu_acts = ops_emulator.run_ops(tensors, ops, x, bf16=True)
    net = network.CompiledNet(plan, h, w, B, layout=layout, fuse_dw=fuse)
    for impl in ((0,) if fuse else (1, 0)):
        heads = net.forward(x.cuda(), gemm_impl=impl)
        torch.cuda.synchronize()
        helpers.assert_taps_match_emulation(net, ops, emu_acts, B, f'impl {impl}')
        for hg, he in zip(heads, emu_heads):
            assert float((hg.cpu() - he).abs().max()) < 5e-2


def test_fields_match_fp32_pytorch_full_size():
    """BASELINE size: 641x641 (41x41 fields), batch 4, vs fp32 PyTorch (no TF32) on the same GPU."""
    shell = net_oracle.make_shell('shufflenetv2k16', seed=2)
    plan = network.plan_from_shell(shell)
    net = network.CompiledNet(plan, 641, 641, 4)
    x = torch.randn(4, 3, 641, 641, generator=torch.Generator().manual_seed(1)).cuda()
    heads = net.forward(x)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        ref = shell.cuda()(x)
    for hg, hr in zip(heads, ref):
        assert hg.shape == hr.shape == (4, hr.shape[1], hr.shape[2], 41, 41)
        err = float((hg - hr).abs().max())
        assert err < FIELD_TOL_REL * float(hr.std()) + 1e-3, err


def test_fused_depthwise_gemm_equals_two_kernels_bitwise():
    """k_dw_gemm writes the depthwise result as bf16 into the GEMM's A operand exactly as the standalone depthwise
    kernel writes it to HBM, and both GEMMs accumulate the same K blocks in the same order: the fields of the fused
    and the two-kernel schedules are identical bit for bit -- at a size with partial edge tiles in both directions,
    many tiles per CTA (ring wrap-around) and batch > 1, for the k16 (N <= 192: one column block per patch; above:
    two) and k30 (N = 256 / 512: two / three column blocks) channel widths."""
    for base, heads in (('shufflenetv2k16', ((17, 1, 1, 1), (19, 1, 2, 2))), ('shufflenetv2k30', ((17, 1, 1, 1), (19, 1, 2, 2)))):
        plan = network.random_plan(base, heads=heads, seed=7)
        B, H, W = 5, 337, 401
        x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(12)).cuda()
        fused = network.CompiledNet(plan, H, W, B, fuse_dw=True)
        plain = network.CompiledNet(plan, H, W, B, fuse_dw=False)
        assert any(o['kind'] == 'dw_conv1x1' for o in fused.op_desc) and not any(o['kind'] == 'dw_conv1x1' for o in plain.op_desc)
        hf = [t.clone() for t in fused.forward(x)]
        hp = [t.clone() for t in plain.forward(x)]
        torch.cuda.synchronize()
        for a, b in zip(hf, hp):
            assert torch.isfinite(a).all()
            assert torch.equal(a, b), float((a - b).abs().max())
        # every stage output too (the tensors the fused ops scatter into)
        for (tf, lf), (tp, lp) in zip(fused.info['block_outputs'], plain.info['block_outputs']):
            np.testing.assert_array_equal(fused.tap(tf, B)[..., lf.cols()], plain.tap(tp, B)[..., lp.cols()])
        fused.close(); plain.close()


def test_linearity_property_of_conv_path():
    """size-independent property: with ReLU-free positive scaling, fields scale consistently --
    forward(x) is deterministic and batch-position independent (image b alone == image b in a batch)."""
    plan = network.random_plan('shufflenetv2k16', seed=4)
    net = network.CompiledNet(plan, 161, 161, 8)
    x = torch.randn(8, 3, 161, 161, generator=torch.Generator().manual_seed(2)).cuda()
    full = [h.clone() for h in net.forward(x)]
    again = [h.clone() for h in net.forward(x)]
    for a, b in zip(full, again):
        assert torch.equal(a, b)
    for b in (0, 5, 7):
        one = net.forward(x[b:b + 1].contiguous())
        for hf, ho in zip(full, one):
            assert torch.equal(hf[b], ho[0])


def test_predictor_end_to_end_host_buffers():
    """Predictor.batch on host images: CUDA decode of the network's fields == oracle decode of the same fields."""
    plan = network.random_plan('shufflenetv2k16', seed=0)
    net = network.CompiledNet(plan, 321, 321, 4)
    pred = predictor.Predictor(net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    imgs = torch.randn(4, 3, 321, 321, generator=torch.Generator().manual_seed(3)).pin_memory()
    res = pred.batch(imgs)
    assert len(res) == 4
    cif, caf = [h.cpu().numpy() for h in net.forward(imgs.cuda())]
    sk = np.asarray(constants.COCO_PERSON_SKELETON, dtype=np.int64) - 1
    p = oc.default_params(seed_sort_stable=1)
    for b in range(4):
        oa, _ = oc.decode(cif[b], 16, caf[b], 16, sk, 17, params=p)
        helpers.assert_annotations_close(res[b][0].numpy(), oa, f'image {b}')


def test_pipelined_batches_equal_sequential():
    """Predictor.batches (H2D / compute overlap, double-buffered results) yields what Predictor.batch yields."""
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=0.0)
    net = network.CompiledNet(plan, 161, 161, 3)
    pred = predictor.Predictor(net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    g = torch.Generator().manual_seed(5)
    hosts = [torch.randn(3, 3, 161, 161, generator=g).pin_memory() for _ in range(5)]
    want = [pred.batch(h) for h in hosts]
    got = list(pred.batches(iter(hosts)))
    assert len(got) == len(want) == 5
    for rw, rg in zip(want, got):
        for (aw, iw), (ag, ig) in zip(rw, rg):
            assert torch.equal(aw, ag) and torch.equal(iw, ig)


@pytest.mark.parametrize('name,size,batch', [('resnet18', 161, 1), ('resnet50', 129, 2)])
def test_resnet_implicit_gemm_matches_emulation_and_fp32(name, size, batch):
    """configs[0] (resnet18, 161x161, single image) and the resnet50 family: 3x3 / strided convs as wgmma
    implicit GEMMs with the fused residual epilogue, per op vs the bf16 emulation and end-to-end vs fp32 PyTorch."""
    shell = net_oracle.make_shell(name, seed=4)
    plan = network.plan_from_shell(shell)
    x = torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(6))
    tensors, ops, _ = network.build_ops(plan, size, size)
    emu_heads, emu_acts = ops_emulator.run_ops(tensors, ops, x, bf16=True)
    net = network.CompiledNet(plan, size, size, batch)
    for impl in (1, 0):
        net.forward(x.cuda(), gemm_impl=impl)
        torch.cuda.synchronize()
        helpers.assert_taps_match_emulation(net, ops, emu_acts, batch, f'{name} impl {impl}')
    with torch.no_grad():
        want = shell(x)
    # vs fp32 PyTorch: bf16 rounding through 21 / 54 layers (resnet50 with randomised BN statistics needs the wider
    # bound); the per-op checks above are the tight ones
    tol = 8e-2 if name == 'resnet50' else FIELD_TOL_REL
    for hg, hw_ in zip(net.forward(x.cuda()), want):
        assert hg.shape == hw_.shape
        err = (hg.cpu() - hw_).abs()
        assert float(err.max()) < tol * float(hw_.std()) + 1e-3
        assert float(err.mean()) < 1e-2 * float(hw_.std())


def test_k30_wholebody_network_and_decode():
    """BASELINE configs[3]: shufflenetv2k30 + wholebody heads (F=133, C=160; 1945 head channels in one GEMM,
    2048-wide stage-4 GEMMs) per op vs the bf16 emulation, fields vs fp32 PyTorch, then the Predictor end to end
    (the decoder handle sized for 133 keypoints / 160 connections) against the oracle decoder on the same fields."""
    shell = net_oracle.make_shell('shufflenetv2k30', n_keypoints=133, n_connections=160, seed=3)
    plan = network.plan_from_shell(shell)
    h, w, B = 129, 161, 2
    x = torch.randn(B, 3, h, w, generator=torch.Generator().manual_seed(8))
    tensors, ops, _ = network.build_ops(plan, h, w)
    emu_heads, emu_acts = ops_emulator.run_ops(tensors, ops, x, bf16=True)
    net = network.CompiledNet(plan, h, w, B)
    heads = net.forward(x.cuda())
    torch.cuda.synchronize()
    helpers.assert_taps_match_emulation(net, ops, emu_acts, B, 'k30 wholebody')
    with torch.no_grad():
        want = shell(x)
    for hg, hw_ in zip(heads, want):
        assert hg.shape == hw_.shape
        err = (hg.cpu() - hw_).abs()
        assert float(err.max()) < 8e-2 * float(hw_.std()) + 1e-3      # 100 bf16 layers
        assert float(err.mean()) < 1e-2 * float(hw_.std())
    skeleton = constants.wholebody_skeleton()
    pred = predictor.Predictor(net, constants.WHOLEBODY_N_KEYPOINTS, skeleton)
    res = pred.batch(x.pin_memory())
    cif, caf = [t.cpu().numpy() for t in net.forward(x.cuda())]
    sk = np.asarray(skeleton, dtype=np.int64) - 1
    p = oc.default_params(seed_sort_stable=1)
    for b in range(B):
        oa, _ = oc.decode(cif[b], 16, caf[b], 16, sk, constants.WHOLEBODY_N_KEYPOINTS, params=p)
        helpers.assert_annotations_close(res[b][0].numpy(), oa, f'k30 wholebody image {b}')


def test_raw_uint8_images_equal_normalised_float_images():
    """SURVEY 8f rank 2 (GPU preprocessing): the stem applies ToTensor + Normalize (transforms/__init__.py:26-33)
    on load; fields and annotations are identical, bit for bit, to the float path fed with the same normalisation
    done by torch on the host."""
    plan = network.random_plan('shufflenetv2k16', seed=0)
    B, H, W = 3, 193, 161
    net = network.CompiledNet(plan, H, W, B)
    g = torch.Generator().manual_seed(11)
    raw = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    mean = torch.tensor(network.CompiledNet.IMAGE_MEAN, dtype=torch.float32)
    std = torch.tensor(network.CompiledNet.IMAGE_STD, dtype=torch.float32)
    normalised = ((raw.permute(0, 3, 1, 2).to(torch.float32) / 255.0) - mean.view(1, 3, 1, 1)) / std.view(1, 3, 1, 1)
    want = [t.clone() for t in net.forward(normalised.contiguous().cuda())]
    got = net.forward_uint8(raw.cuda())
    for tg, tw in zip(got, want):
        assert torch.equal(tg, tw)
    pred = predictor.Predictor(net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    res_f = pred.batch(normalised.contiguous().pin_memory())
    res_u = pred.batch(raw.pin_memory())
    for (af, idf), (au, idu) in zip(res_f, res_u):
        assert torch.equal(af, au) and torch.equal(idf, idu)
    with pytest.raises(RuntimeError):
        net.forward_uint8(raw[:, :10].cuda())


@pytest.mark.parametrize('up', [2, 3])
def test_upsampled_heads_pixelshuffle_in_the_epilogue(up):
    """SURVEY.md 8f rank 4: upsample_stride > 1 heads (heads.py:307-343).  The heads GEMM writes PixelShuffle(up) +
    crop + the CompositeField4 eval ops straight from its epilogue; checked against plain torch ops (conv as a matmul
    on the same bf16-rounded operands, torch.nn.PixelShuffle, the reference's crop, sigmoid / index add / softplus)."""
    rng = np.random.default_rng(up)
    c_in, h, w, B = 136, 9, 13, 3
    heads_spec = ((5, 1, 1, 1), (4, 1, 2, 2))         # a CIF-like and a CAF-like head
    heads = []
    for nf, nconf, nvec, nsc in heads_spec:
        ncomp = 1 + nconf + 2 * nvec + nsc
        heads.append({'w': (rng.standard_normal((nf * ncomp * up * up, c_in)) / np.sqrt(c_in)).astype(np.float32),
                      'b': (rng.standard_normal(nf * ncomp * up * up) * 0.3).astype(np.float32),
                      'n_fields': nf, 'n_comp': ncomp, 'upsample': up,
                      'ops': network.head_ops(nconf, nvec, nsc, (True,) * nvec), 'stride': 16 // up})
    plan = {'kind': 'heads_only', 'c_in': c_in, 'heads': heads}
    net = network.CompiledNet(plan, h, w, B)
    feat = rng.standard_normal((B, h, w, c_in)).astype(np.float32)
    got = [t.clone().cpu() for t in net.forward_features(feat)]

    def bf16(a):
        return torch.from_numpy(a).to(torch.bfloat16).to(torch.float64)
    x = bf16(feat).permute(0, 3, 1, 2)                                   # [B, C, h, w]
    low, high = (up - 1) // 2, int(np.ceil((up - 1) / 2.0))
    for hd, g in zip(heads, got):
        y = torch.einsum('bchw,nc->bnhw', x, bf16(hd['w'])) + torch.from_numpy(hd['b']).double().view(1, -1, 1, 1)
        y = torch.nn.PixelShuffle(up)(y)
        y = y[:, :, low:y.shape[2] - high, low:y.shape[3] - high]
        H2, W2 = y.shape[2], y.shape[3]
        assert (H2, W2) == (h * up - low - high, w * up - low - high)
        y = y.reshape(B, hd['n_fields'], hd['n_comp'], H2, W2).clone()
        xs = torch.arange(W2, dtype=torch.float64).view(1, 1, 1, W2)
        ys = torch.arange(H2, dtype=torch.float64).view(1, 1, H2, 1)
        for c, op in enumerate(hd['ops']):
            if op == network.OP_SIGMOID:
                y[:, :, c] = torch.sigmoid(y[:, :, c])
            elif op == network.OP_ADD_X:
                y[:, :, c] += xs
            elif op == network.OP_ADD_Y:
                y[:, :, c] += ys
            elif op == network.OP_SOFTPLUS:
                y[:, :, c] = torch.nn.functional.softplus(y[:, :, c])
        assert tuple(g.shape) == tuple(y.shape)
        assert float((g.double() - y).abs().max()) < 2e-4
    net.close()
