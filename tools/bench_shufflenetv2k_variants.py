"""Time shufflenetv2k16 with --shufflenetv2k-stage4-dilation 2 (stride 8: 81 x 81 fields at 641 px) on the GPU: the
compiled forward and its per-op-kind split, the dilated depthwise launches (the dilation-2 mode of the TMA kernel) in
algorithmic GB/s next to the undilated stride-1 5x5 launches of the same net and next to the same dilated ops on the
generic kernel (gemm_impl = 1 routes every depthwise op there), forward + CifCaf decode + fetch through
`predictor.Predictor` on planted poses, and the stock PyTorch forward of the same architecture (fp32, and bf16
channels_last).

The compiled model is network.random_plan('shufflenetv2k16', stage4_dilation=2) with the CocoKp heads calibrated as
bench.py calibrates its plans.  The stock forward runs the test mirror of the reference's module
(tests/shufflenetv2k_models.py) with seeded weights: the same shapes, other weights.  A random net emits no poses, so
the decode inside each timed step runs on planted fields (synth.make_fields, Poisson(4)+1 people per image, one
81 x 81 field set per image).

    python tools/bench_shufflenetv2k_variants.py --out DIR [--size 641] [--batch 64] [--steps 20] [--warmup 5]

Writes DIR/bench_shufflenetv2k_variants.json with the card name, its power limit and SM clock (nvidia-smi, same run)."""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import shufflenetv2k_models as sm                      # noqa: E402
from openpifpaf_b200 import constants, network, predictor, synth   # noqa: E402

KINDS = ((0, 'input_conv'), (1, 'gemm'), (2, 'dwconv'), (3, 'fused'))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, max_clock, clock = (v.strip() for v in q.split(','))
    return {'name': name, 'power_limit': power, 'max_sm_clock': max_clock, 'sm_clock': clock}


def timed(fn, steps, warmup):
    """ms per call: host clock around `steps` calls that each end in a device synchronise"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1000.0 / steps


def event_ms(fn, steps, warmup):
    """ms per call from CUDA events around `steps` back-to-back calls"""
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def dw_rates(ops, ms, nbytes, select):
    """summed ms and algorithmic GB/s (input + output of the real channels, as pifpaf_net_forward_timed counts them)
    of the depthwise ops `select` picks"""
    idx = [i for i, o in enumerate(ops) if o['kind'] == 'dwconv' and select(o)]
    t = float(sum(ms[i] for i in idx))
    b = float(sum(nbytes[i] for i in idx))
    return {'launches': len(idx), 'ms': t, 'gb_per_s': b / 1e6 / t if t > 0 else None}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', required=True, help='directory for bench_shufflenetv2k_variants.json')
    ap.add_argument('--size', type=int, default=641)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_shufflenetv2k_variants.py needs a CUDA device')
    size, batch, steps, warmup = args.size, args.batch, args.steps, args.warmup
    dev = torch.device('cuda', 0)
    out = {'card': card(), 'model': 'shufflenetv2k16, stage4_dilation 2, CocoKp heads', 'size': size, 'batch': batch,
           'steps': steps, 'warmup': warmup, 'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32}

    heads = ((constants.COCO_N_KEYPOINTS, 1, 1, 1), (len(constants.COCO_PERSON_SKELETON), 1, 2, 2))
    plan = network.random_plan('shufflenetv2k16', heads=heads, seed=0, confidence_bias=-2.5, stage4_dilation=2)
    network.calibrate_random_heads(plan, size=min(size, 641), batch=2)
    net = network.CompiledNet(plan, size, size, batch)
    out['fields'] = [net.heads[0]['h'], net.heads[0]['w']]
    out['gflop_per_image'] = net.flops_per_image / 1e9
    tensors, ops, _ = network.build_ops(plan, size, size)
    assert len(ops) == net.num_ops

    images = torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(1))
    x = images.to(dev)
    out['compiled_forward_ms'] = event_ms(lambda: net.forward(x), steps, warmup)
    ms, kind, _, nbytes = net.forward_timed(x)
    ms, kind, nbytes = ms.copy(), kind.copy(), nbytes.copy()        # bytes of the whole batch
    out['compiled_forward_ms_by_kind'] = {name: float(ms[kind == k].sum()) for k, name in KINDS}
    # the GEMMs of stage 4, conv5 and the heads, which read the stride-8 map (four times the pixels of the stride-16
    # net's)
    out['gemm_ms_at_field_size'] = float(sum(ms[i] for i, o in enumerate(ops) if o['kind'] in ('conv1x1', 'heads') and
                                             list(tensors[o['in']][:2]) == out['fields']))
    dilated = dw_rates(ops, ms, nbytes, lambda o: o.get('dilation', 1) == 2)
    undilated = dw_rates(ops, ms, nbytes, lambda o: o.get('dilation', 1) == 1 and o['stride'] == 1 and o['kernel'] == 5)
    net.forward_timed(x, gemm_impl=1)                   # warm the generic kernels
    ms1, _, _, _ = net.forward_timed(x, gemm_impl=1)
    generic = dw_rates(ops, ms1.copy(), nbytes, lambda o: o.get('dilation', 1) == 2)
    out['dwconv_5x5_dilated2_tma'] = dilated
    out['dwconv_5x5_stride1_undilated_tma'] = undilated
    out['dwconv_5x5_dilated2_generic'] = generic
    out['dilated_tma_speedup_over_generic'] = generic['ms'] / dilated['ms']

    pred = predictor.Predictor(net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    h, w = net.heads[0]['h'], net.heads[0]['w']
    items = [synth.make_fields('cocokp', h, w, None, 77 * 1000 + b) for b in range(batch)]
    cif = torch.from_numpy(np.stack([it['cif'] for it in items])).to(dev)
    caf = torch.from_numpy(np.stack([it['caf'] for it in items])).to(dev)
    pred.decode_fields_override = (cif, 8, caf, 8)
    out['planted_people'] = int(sum(it['n_planted'] for it in items))

    def compiled_e2e():
        pred.batch_device(x)
        return pred.decoder.fetch()
    out['compiled_forward_decode_fetch_ms'] = timed(compiled_e2e, steps, warmup)
    out['annotations'] = int(sum(a.shape[0] for a, _ in compiled_e2e()))
    out['images_per_s_compiled'] = batch * 1000.0 / out['compiled_forward_decode_fetch_ms']
    pred.close()

    ref32 = sm.make_pose_shell('dil2', 'shufflenetv2k16', seed=0).to(dev)
    ref16 = copy.deepcopy(ref32).to(dtype=torch.bfloat16, memory_format=torch.channels_last)
    x16 = x.to(dtype=torch.bfloat16, memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True
    for label, model, inp in (('fp32', ref32, x), ('bf16_channels_last', ref16, x16)):
        with torch.no_grad():
            out[f'stock_forward_{label}_ms'] = event_ms(lambda: model(inp), steps, warmup)
    out['card_after'] = card()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'bench_shufflenetv2k_variants.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
