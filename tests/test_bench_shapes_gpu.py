"""GPU: the networks bench.py and tools/bench_*.py time, built as they build them and run at the shapes they time
(64 images of 641 x 641, the 32-image shard, C3 and C4), checked op by op against the float64 reference.

Each case runs one forward, then every op of build_ops teacher-forced (kernel_refs.op_ref on the tensors the GPU fed
it) at kernel_refs.op_positions: image borders, tile corners of the last image, the first and last 128-row GEMM tiles,
the pixels around byte 2^31 of the 2.5 GB stage-2 entry tensor t_c, and 4096 seeded pixels over the whole batch.
Tensors are tapped one at a time (the op's inputs and outputs) and freed, and every real channel of every tensor is
checked finite over the whole batch.  Defects that only exist at this scale -- persistent CTAs walking 16x more tiles,
large tile and work indices, the last image's last tile, byte offsets past 2^31 -- are what these cases look for."""
import resource
import time

import numpy as np
import pytest
import torch

import bench
import helpers
import kernel_refs as kr
from openpifpaf_b200 import constants, decoder, network, predictor, synth
from oracle import cifcaf as oc

pytestmark = pytest.mark.gpu

SIZE = 641


def peak_rss_gb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20


def bench_plan(name, **kw):
    """bench.make_plan calibrated as bench.build_predictor calibrates it (kw: bench.make_plan's config overrides)"""
    cfg = dict(bench.CONFIGS[name], **kw)
    plan = bench.make_plan(cfg)
    network.calibrate_random_heads(plan, size=min(cfg['size'], 641), batch=2)
    return plan


def dil2_plan():
    """tools/bench_shufflenetv2k_variants.py: k16 with stage-4 dilation 2, CocoKp heads calibrated as bench.py does"""
    K = synth.WORKLOADS['cocokp'][0]
    heads = ((K, 1, 1, 1), (len(synth.skeleton_for('cocokp')), 1, 2, 2))
    plan = network.random_plan('shufflenetv2k16', heads=heads, seed=0, confidence_bias=-2.5, stage4_dilation=2)
    network.calibrate_random_heads(plan, size=641, batch=2)
    return plan


def mnv2_plan():
    """tools/bench_mobilenetv2.py"""
    import mobilenetv2_models as mm
    return network.plan_from_shell(mm.make_pose_shell(seed=0))


def cocodet_plan():
    """tools/bench_det.py: resnet18-cocodet (upsample-2 CifDet heads), head calibrated as there"""
    import det_models
    shell = det_models.make_variant_shell('cocodet', seed=0)
    det_models.calibrate_det_head(shell)
    return network.plan_from_shell(shell)


# case -> (plan factory, batch, input size (h, w) or None for the capacity, env, gemm_impl, uint8 stem)
CASES = {
    'C0': (lambda: bench_plan('C0'), 64, None, {}, 0, False),
    'C0-u8': (lambda: bench_plan('C0'), 64, None, {}, 0, True),
    'C0-unfused': (lambda: bench_plan('C0'), 64, None, {'PIFPAF_FUSE_PW_DW': '0'}, 0, False),
    'C0-lanes': (lambda: bench_plan('C0'), 64, None, {'PIFPAF_FUSE_PW_DW': '0', 'PIFPAF_GEMM_TMA_STORE': '0'}, 0, False),
    'C0-simt': (lambda: bench_plan('C0'), 64, None, {'PIFPAF_FUSE_PW_DW': '0'}, 1, False),
    'C2': (lambda: bench_plan('C2'), 32, None, {}, 0, False),
    'C3': (lambda: bench_plan('C3'), 16, None, {}, 0, False),
    'C4': (lambda: bench_plan('C4'), 8, None, {}, 0, False),
    # tools/bench_sizes.py: k16 compiled at 64 x 641 x 641, run on the 641 x 481 tight canvas
    'sizes': (lambda: network.random_plan('shufflenetv2k16', seed=0), 64, (641, 481), {}, 0, False),
    'mnv2': (mnv2_plan, 64, None, {}, 0, False),
    'dil2': (dil2_plan, 64, None, {}, 0, False),
    'cocodet': (cocodet_plan, 64, None, {}, 0, False),
}
CAPACITY = {'C4': 801}


def reads_and_writes(o):
    """the tensors op o of build_ops reads and writes"""
    ts = {o['in']} if o['kind'] != 'input_conv' else set()
    ts |= {pc[2] for pc in o['pieces']} if 'pieces' in o else ({o['out']} if 'out' in o else set())
    ts |= {o[k] for k in ('residual', 'shuffle_src') if o.get(k, -1) >= 0}
    return ts


def runs(cols):
    """sorted column indices -> [(first, end)] of their contiguous runs"""
    cuts = np.flatnonzero(np.diff(cols) != 1) + 1
    return [(int(r[0]), int(r[-1]) + 1) for r in np.split(cols, cuts) if len(r)]


def check_ops_sampled(net, ops, tensors, images, fields, B, label):
    """every op of ops (build_ops at the net's current size) at op_positions against op_ref, on taps of the forward
    that produced `fields` (host arrays); -> {kind: worst err / bound}"""
    written = {}
    for o in ops:
        for t, c0, c1 in kr.written_columns(o, tensors):
            written.setdefault(t, np.zeros(tensors[t][2], dtype=bool))[c0:c1] = True
    cache, seen, worst = {}, set(), {}
    for i, o in enumerate(ops):
        need = reads_and_writes(o)
        for t in [t for t in cache if t not in need]:
            del cache[t]
        for t in sorted(need - set(cache)):
            cache[t] = net.tap(t, B)
            if t not in seen:
                seen.add(t)
                real = np.flatnonzero(written.get(t, []))
                for c0, c1 in runs(real):
                    assert np.isfinite(cache[t][..., c0:c1]).all(), (label, 'tensor', t, 'columns', c0, c1)
        pos = kr.op_positions(o, tensors, B, seed=i)
        kind, r = kr.op_ref(o, cache, fields, images, B, positions=pos)
        worst[kind] = max(worst.get(kind, 0.0), r)
        big = [(t, m) for t in sorted(need) for m in kr.crossing_rows(B * tensors[t][0] * tensors[t][1], tensors[t][2])]
        print(f'  {label} op {i:3d} {kind:18s} {len(pos):6d} positions  err/bound {r:.3f}'
              + ''.join(f'  t{t} crossing row {m} = image {m // (tensors[t][0] * tensors[t][1])} pixel '
                        f'{m // tensors[t][1] % tensors[t][0]},{m % tensors[t][1]}' for t, m in big))
        assert r <= 1.0, f'{label} op {i} ({kind}): err / bound = {r:.3g}'
    cache.clear()
    return worst


def check_head_images(net, ops, fields, B, label):
    """every head-output value of images 0, B/2 and B-1 against heads_ref on the tapped feature map, and every head
    output finite over the whole batch"""
    o = next(o for o in ops if o['kind'] == 'heads')
    idx = sorted({0, B // 2, B - 1})
    feat = net.tap(o['in'], B)[idx][..., :o['k_cols']]
    refs = kr.heads_ref(feat, kr.bf16_round(o['w']), o['b'], o['n_fields'], o['n_comp'], o['ops'], o['upsample'])
    worst = 0.0
    for hb, (r, bd) in zip(fields, refs):
        assert np.isfinite(hb).all(), label
        worst = max(worst, kr.worst_ratio(hb[idx], r, bd))
    assert worst <= 1.0, f'{label} heads of images {idx}: err / bound = {worst:.3g}'
    return worst


@pytest.mark.parametrize('case', list(CASES))
def test_bench_shape_ops_against_float64(case, monkeypatch):
    t0 = time.perf_counter()
    make, B, size, env, impl, u8 = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cap = CAPACITY.get(case, SIZE)
    plan = make()
    net = network.CompiledNet(plan, cap, cap, B)
    H, W = size or (cap, cap)
    if size is not None:
        net.set_input_size(H, W)
    tensors, ops, _ = network.build_ops(plan, H, W)
    assert [tuple(s) for s in tensors] == [tuple(s) for s in net.tensor_shapes]
    g = torch.Generator().manual_seed(64 + len(case))
    if u8:
        raw = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
        images = kr.normalise_u8(raw.numpy(), net.IMAGE_MEAN, net.IMAGE_STD).transpose(0, 3, 1, 2)
        fields = [t.cpu().numpy() for t in net.forward_uint8(raw.cuda(), gemm_impl=impl)]
    else:
        x = torch.randn((B, 3, H, W), generator=g)
        images = x.numpy()
        fields = [t.cpu().numpy() for t in net.forward(x.cuda(), gemm_impl=impl)]
    torch.cuda.synchronize()
    worst = check_ops_sampled(net, ops, tensors, images, fields, B, case)
    worst['heads (images 0, B/2, B-1)'] = check_head_images(net, ops, fields, B, case)
    if case == 'C0':
        # bench.py's roofline times forward_timed: the timed schedule computes the fields of forward, bit for bit
        net.forward_timed(torch.from_numpy(images).cuda())
        torch.cuda.synchronize()
        for got, want in zip(net._head_views(B), fields):
            assert np.array_equal(got.cpu().numpy(), want), 'forward_timed'
    net.close()
    print(f'{case}: {B} x {H} x {W}, {time.perf_counter() - t0:.1f} s, peak host RSS {peak_rss_gb():.2f} GB')
    for k in sorted(worst):
        print(f'  {case:10s} {k:28s} {worst[k]:.3f}')


def test_overlapped_predictor_at_bench_size(monkeypatch):
    """Predictor(overlap_decode=True) at 64 x 641 (the reserve policy keeps every SM for the forward at 64 images),
    three steps of distinct images: the annotations and fields of the sequential predictor, bit for bit"""
    monkeypatch.setattr(decoder.NMSKeypoints, '_instance_threshold', 0.0)
    plan = network.random_plan('shufflenetv2k16', seed=0, confidence_bias=-2.0)
    for hd in plan['heads']:
        hd['w'] = hd['w'] * np.float32(0.06)
    B = 64
    g = torch.Generator().manual_seed(640)
    hosts = [torch.randn(B, 3, SIZE, SIZE, generator=g).pin_memory() for _ in range(3)]
    seq_net = network.CompiledNet(plan, SIZE, SIZE, B)
    seq = predictor.Predictor(seq_net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    want, want_fields = [], []
    for hst in hosts:
        want.append(seq.batch(hst))
        torch.cuda.synchronize()
        want_fields.append([t.cpu() for t in seq_net.forward(hst.cuda())])
        torch.cuda.synchronize()
    seq.close()
    ovl_net = network.CompiledNet(plan, SIZE, SIZE, B)
    ovl = predictor.Predictor(ovl_net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON, overlap_decode=True)
    dev = [h.cuda() for h in hosts]
    torch.cuda.synchronize()
    got, got_fields, outstanding = [], [], 0
    with torch.cuda.stream(ovl.stream):
        for d in dev:
            ovl.batch_device(d)
            got_fields.append([t.clone() for t in ovl_net._head_views(B)])
            ovl.decoder.fetch_begin(stream=ovl.result_stream())
            outstanding += 1
            if outstanding == 2:
                got.append(ovl.decoder.fetch_end())
                outstanding -= 1
        got.append(ovl.decoder.fetch_end())
        ovl.join()
    torch.cuda.synchronize()
    ovl.close()
    n_ann = []
    for step, (rw, rg) in enumerate(zip(want, got)):
        assert len(rw) == len(rg) == B
        for (aw, iw), (ag, ig) in zip(rw, rg):
            assert torch.equal(aw, ag) and torch.equal(iw, ig), step
        for a, b in zip(got_fields[step], want_fields[step]):
            assert torch.equal(a.cpu(), b), step
        n_ann.append(sum(int(aw.shape[0]) for aw, _ in rw))
    print('overlap 64 x 641 annotations per step', n_ann)
    assert len(got) == 3 and min(n_ann) > 0


@pytest.mark.parametrize('overlap', [False, True])
@pytest.mark.parametrize('name', ['C3', 'C5'])
def test_bench_decode_path_on_planted_fields(name, overlap):
    """bench.timed_steps' decode: bench.planted_fields through the bench predictor's decode_fields_override, three
    decode_batch_async calls before one fetch; every image against the oracle decoder (DESIGN section 2 contract)"""
    cfg = bench.CONFIGS[name]
    B = cfg['batch']
    _, net, pred = bench.build_predictor(cfg, B, 0, overlap)
    f = bench.planted_fields(cfg, B)
    dev = torch.device('cuda', 0)
    pred.decode_fields_override = (torch.from_numpy(f['cif']).to(dev), 16, torch.from_numpy(f['caf']).to(dev), 16)
    images = torch.randn((B, 3, cfg['size'], cfg['size']), generator=torch.Generator().manual_seed(5)).to(dev)
    for _ in range(3):
        pred.batch_device(images)
    pred.join()
    res = pred.decoder.fetch(stream=pred.result_stream())
    torch.cuda.synchronize()
    pred.close()
    K = synth.WORKLOADS[cfg['workload']][0]
    sk = np.asarray(synth.skeleton_for(cfg['workload']), dtype=np.int64) - 1
    p = oc.default_params(seed_sort_stable=1)
    assert len(res) == B
    n = 0
    for b in range(B):
        want, _ = oc.decode(f['cif'][b], 16, f['caf'][b], 16, sk, K, params=p)
        helpers.assert_annotations_close(res[b][0].cpu().numpy(), want, f'{name} image {b}')
        n += len(want)
    print(name, 'overlap' if overlap else 'sequential', B, 'images', n, 'annotations')
    assert n > 0
