"""Time the MobileNetV2 pose model (reference basenetworks.py:407-417 with the CocoKp heads) on the GPU: the compiled
forward alone, forward + CifCaf decode + fetch through `predictor.Predictor` on planted poses, and the stock PyTorch
forward of the same Shell (fp32, and bf16 channels_last).  Also reports the algorithmic bytes of every op kind
(input + output of every conv, real channels, computed from shapes) and the card the numbers were taken on.

The model is the test mirror of the reference's module (tests/mobilenetv2_models.py) with seeded from-scratch weights
and random BatchNorm statistics.  A random net emits no poses, so the decode inside each timed step runs on planted
fields (synth.make_fields, Poisson(4)+1 people per image, one 21 x 21 field set per image as at 641 px).

    python tools/bench_mobilenetv2.py --out DIR [--size 641] [--batch 64] [--steps 20] [--warmup 5]

Writes DIR/bench_mobilenetv2.json with the card name, its power limit and max SM clock (nvidia-smi, same run)."""
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
import mobilenetv2_models as mm                       # noqa: E402
from openpifpaf_b200 import network, predictor, synth   # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (v.strip() for v in q.split(','))
    return {'name': name, 'power_limit': power, 'max_sm_clock': clock}


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


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', required=True, help='directory for bench_mobilenetv2.json')
    ap.add_argument('--size', type=int, default=641)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mobilenetv2.py needs a CUDA device')
    size, batch, steps, warmup = args.size, args.batch, args.steps, args.warmup
    dev = torch.device('cuda', 0)
    out = {'card': card(), 'model': 'mobilenetv2 + CocoKp heads', 'size': size, 'batch': batch, 'steps': steps,
           'warmup': warmup, 'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32}

    shell = mm.make_pose_shell(seed=0)
    plan = network.plan_from_shell(shell)
    tensors, ops, _ = network.build_ops(plan, size, size)
    out['gflop_per_image'] = mm.flops(tensors, ops) / 1e9
    out['algorithmic_mb_per_image'] = {k: v / 1e6 for k, v in mm.algorithmic_bytes(tensors, ops).items()}
    out['algorithmic_mb_per_image']['total'] = sum(mm.algorithmic_bytes(tensors, ops).values()) / 1e6

    images = torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(1))
    x = images.to(dev)
    pred = predictor.from_shell(shell, size, size, batch)
    out['compiled_forward_ms'] = event_ms(lambda: pred.net.forward(x), steps, warmup)
    ms, kind, _, _ = pred.net.forward_timed(x)
    out['compiled_forward_ms_by_kind'] = {name: float(ms[kind == k].sum()) for k, name in
                                          ((0, 'input_conv'), (1, 'gemm'), (2, 'dwconv'))}
    ops_ms = {'conv': 0.0, 'conv residual': 0.0, 'dwconv': 0.0}
    ab = {'conv': 0.0, 'conv residual': 0.0, 'dwconv': 0.0}
    for o, t in zip(ops, ms):
        if o['kind'] in ('input_conv', 'heads'):
            continue
        k = 'conv residual' if o['kind'] == 'conv' and o['residual'] >= 0 else o['kind']
        ops_ms[k] += float(t)
        ab[k] += mm.algorithmic_bytes(tensors, [o], batch)[k]
    out['per_kind_gb_per_s'] = {k: ab[k] / 1e6 / ops_ms[k] for k in ops_ms}

    h, w = pred.net.heads[0]['h'], pred.net.heads[0]['w']
    items = [synth.make_fields('cocokp', h, w, None, 77 * 1000 + b) for b in range(batch)]
    cif = torch.from_numpy(np.stack([it['cif'] for it in items])).to(dev)
    caf = torch.from_numpy(np.stack([it['caf'] for it in items])).to(dev)
    pred.decode_fields_override = (cif, 32, caf, 32)
    out['planted_people'] = int(sum(it['n_planted'] for it in items))

    def compiled_e2e():
        pred.batch_device(x)
        return pred.decoder.fetch()
    out['compiled_forward_decode_fetch_ms'] = timed(compiled_e2e, steps, warmup)
    out['annotations'] = int(sum(a.shape[0] for a, _ in compiled_e2e()))
    out['images_per_s_compiled'] = batch * 1000.0 / out['compiled_forward_decode_fetch_ms']
    pred.close()

    ref32 = shell.to(dev)
    ref16 = copy.deepcopy(ref32).to(dtype=torch.bfloat16, memory_format=torch.channels_last)
    x16 = x.to(dtype=torch.bfloat16, memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True
    for label, model, inp in (('fp32', ref32, x), ('bf16_channels_last', ref16, x16)):
        with torch.no_grad():
            out[f'stock_forward_{label}_ms'] = event_ms(lambda: model(inp), steps, warmup)
    out['card_after'] = card()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'bench_mobilenetv2.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
