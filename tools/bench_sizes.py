"""What running one shufflenetv2k16 net at several input sizes costs, against compiling a net per size.

  compile_ms       CompiledNet(plan, h, w, 64) for a new canvas shape (BN-folded plan given: weight packing and upload,
                   activation buffers for 64 images, every tensor map), host clock around the constructor and a
                   device synchronise; one row per shape, each shape compiled for the first time in the process
  switch_ms        set_input_size on a 641 x 641 net, alternating 641 x 481 and 641 x 641 (host clock: the call is
                   host-only, it enqueues nothing)
  forward_ms       the forward of 64 seeded images (float input, CUDA events, median over reps) on that net at
                   641 x 641 and at 641 x 481, and on a net compiled at exactly 641 x 481, interleaved rep by rep

The card's name, power limit and SM clocks are read in the same run.  Writes DIR/bench_sizes.json and prints it.

    python tools/bench_sizes.py --out DIR [--batch 64] [--reps 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_zoom import card      # noqa: E402

CANVASES = [(641, 481), (481, 641), (641, 433), (433, 641), (641, 369)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import torch
    from openpifpaf_b200 import network
    if not torch.cuda.is_available():
        raise SystemExit('bench_sizes needs a GPU')
    os.makedirs(args.out, exist_ok=True)
    B = args.batch
    res = {'host': card(), 'model': 'shufflenetv2k16 (random init)', 'batch': B}
    plan = network.random_plan('shufflenetv2k16', seed=0)
    torch.cuda.synchronize()

    res['compile_ms'] = {}
    nets = {}
    for h, w in [(641, 641)] + CANVASES[:3]:
        t0 = time.perf_counter()
        nets[(h, w)] = network.CompiledNet(plan, h, w, B)
        torch.cuda.synchronize()
        res['compile_ms'][f'{h}x{w}'] = (time.perf_counter() - t0) * 1e3
    net, exact = nets[(641, 641)], nets[(641, 481)]
    for size in CANVASES[1:3]:
        nets.pop(size).close()

    switches = []
    for i in range(2 * args.reps):
        size = (641, 481) if i % 2 == 0 else (641, 641)
        t0 = time.perf_counter()
        net.set_input_size(*size)
        switches.append((time.perf_counter() - t0) * 1e3)
    res['switch_ms'] = {'median': float(np.median(switches)), 'min': float(np.min(switches)),
                        'max': float(np.max(switches)), 'calls': len(switches)}

    g = torch.Generator().manual_seed(0)
    x_sq = torch.randn((B, 3, 641, 641), generator=g).cuda()
    x_43 = torch.randn((B, 3, 641, 481), generator=g).cuda()
    cases = {'capacity_net_at_641x641': (net, (641, 641), x_sq), 'capacity_net_at_641x481': (net, (641, 481), x_43),
             'net_compiled_at_641x481': (exact, (641, 481), x_43)}
    times = {k: [] for k in cases}
    st = torch.cuda.current_stream()
    for rep in range(args.reps + 3):
        for k, (n, size, x) in cases.items():
            n.set_input_size(*size)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            n.forward(x)
            e1.record(st)
            e1.synchronize()
            if rep >= 3:                     # the first reps warm every shape up
                times[k].append(e0.elapsed_time(e1))
    res['forward_ms'] = {k: {'median': float(np.median(v)), 'min': float(np.min(v)), 'max': float(np.max(v))}
                         for k, v in times.items()}
    # the same fields either way
    net.set_input_size(641, 481)
    a = [t.clone() for t in net.forward(x_43)]
    b = exact.forward(x_43)
    torch.cuda.synchronize()
    res['fields_equal_to_exact_compile'] = all(torch.equal(u, v) for u, v in zip(a, b))
    res['pixels_641x481_over_641x641'] = 481 / 641
    res['host_after'] = card()
    with open(os.path.join(args.out, 'bench_sizes.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
