"""JPEG decode cost: the GPU decoder (pifpaf_jpeg_decode) against Pillow on the host, and Predictor.jpeg_images
against a host decode followed by Predictor.raw_images.

Input: 64 seeded photo-like images (openpifpaf_b200.synth.photo_like_image) at 640 x 480, 4:2:0, quality 90 -- what
the bench's 1700 images/s would read from disk.  Reported: bits per pixel; GPU decode of the batch (CUDA events
around the whole call, per-kernel times from torch.profiler in a separate pass, sync rounds and serial fallbacks);
Pillow decode wall clock on one and on all host cores; end-to-end per-batch time of both routes; the card's name and
power limit and the host's CPU count, read in the same run.  Writes DIR/bench_jpeg.json and prints it.

    python tools/bench_jpeg.py --out DIR [--images 64] [--reps 20]
"""
import argparse
import io
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _pillow_decode(data):
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        return np.asarray(im.convert('RGB')).shape


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = 'nvidia-smi unavailable'
    return {'gpu': q, 'cpu_count': os.cpu_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--images', type=int, default=64)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import torch
    from PIL import Image
    from openpifpaf_b200 import constants, network, predictor, synth
    from openpifpaf_b200 import preprocess as pp
    if not torch.cuda.is_available():
        raise SystemExit('bench_jpeg needs a GPU')
    os.makedirs(args.out, exist_ok=True)
    res = {'host': card()}

    datas = []
    for i in range(args.images):
        b = io.BytesIO()
        Image.fromarray(synth.photo_like_image(480, 640, seed=i)).save(b, 'JPEG', quality=90, subsampling=2)
        datas.append(b.getvalue())
    n_bytes = sum(len(d) for d in datas)
    res['input'] = {'images': args.images, 'size': '640x480', 'subsampling': '4:2:0', 'quality': 90,
                    'bytes': n_bytes, 'bits_per_pixel': 8.0 * n_bytes / (args.images * 640 * 480)}

    # GPU decode: whole call (host parse + staging + kernels) in CUDA events, median over reps
    dec = pp.GpuJpegDecoder(args.images, n_bytes, 640 * 480)
    st = torch.cuda.current_stream()
    for cap in (-1, 0):
        name = 'default_rounds' if cap < 0 else 'serial'
        for _ in range(3):
            dec(datas, max_rounds=cap)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            dec(datas, max_rounds=cap)
            e1.record(st)
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        res[f'gpu_decode_{name}'] = {'ms_median': float(np.median(times)), 'ms_min': float(np.min(times)),
                                     'images_per_s': args.images / (np.median(times) / 1e3), **dec.stats()}
    # host wall clock of the call alone (parse + staging copy enqueue), no synchronise
    t0 = time.perf_counter()
    for _ in range(args.reps):
        dec(datas)
    res['gpu_decode_host_ms_per_call'] = (time.perf_counter() - t0) / args.reps * 1e3
    torch.cuda.synchronize()
    # per kernel, a separate profiled pass
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            dec(datas)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.key.startswith('_ZN') or 'k_jpeg' in ev.key or 'Memcpy' in ev.key or 'Memset' in ev.key:
            name = next((k for k in ('k_jpeg_unstuff_count', 'k_jpeg_unstuff_scan', 'k_jpeg_unstuff_write',
                                     'k_jpeg_subseq_setup', 'k_jpeg_sync', 'k_jpeg_settle', 'k_jpeg_write',
                                     'k_jpeg_dc', 'k_jpeg_idct', 'k_jpeg_color') if k in ev.key), ev.key[:40])
            t = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0)
            kernels[name] = kernels.get(name, 0.0) + t / 5 / 1e3
    res['gpu_kernels_ms_per_batch'] = kernels
    prof.export_chrome_trace(os.path.join(args.out, 'bench_jpeg_trace.json'))

    # Pillow, one core and all cores
    for _ in range(2):
        [_pillow_decode(d) for d in datas]
    t0 = time.perf_counter()
    for _ in range(3):
        [_pillow_decode(d) for d in datas]
    one = (time.perf_counter() - t0) / 3
    ncpu = os.cpu_count()
    with mp.get_context('fork').Pool(ncpu) as pool:
        pool.map(_pillow_decode, datas)
        t0 = time.perf_counter()
        for _ in range(3):
            pool.map(_pillow_decode, datas, chunksize=max(1, len(datas) // (4 * ncpu)))
        allc = (time.perf_counter() - t0) / 3
    res['pillow_1_core'] = {'ms': one * 1e3, 'images_per_s': args.images / one}
    res['pillow_all_cores'] = {'cores': ncpu, 'ms': allc * 1e3, 'images_per_s': args.images / allc}
    res['cores_for_1700_images_per_s'] = 1700 / (args.images / one)

    # end to end: jpeg_images against Pillow decode + raw_images (shufflenetv2k16 random weights, 641 input)
    plan = network.random_plan('shufflenetv2k16', seed=0)
    pred = predictor.Predictor(network.CompiledNet(plan, 641, 641, args.images), constants.COCO_N_KEYPOINTS,
                               constants.COCO_PERSON_SKELETON)
    fill = [(0, 0, 0)] * args.images
    for _ in range(2):
        pred.jpeg_images(datas, fill=fill)
        pred.raw_images([pp.pillow_rgb(d) for d in datas], fill=fill)
    e2e = {'jpeg_images': [], 'pillow_then_raw_images': []}
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pred.jpeg_images(datas, fill=fill)
        torch.cuda.synchronize()
        e2e['jpeg_images'].append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        pred.raw_images([pp.pillow_rgb(d) for d in datas], fill=fill)
        torch.cuda.synchronize()
        e2e['pillow_then_raw_images'].append(time.perf_counter() - t0)
    res['end_to_end_ms_per_batch'] = {k: float(np.median(v) * 1e3) for k, v in e2e.items()}
    pred.close()
    dec.close()
    res['host_after'] = card()
    with open(os.path.join(args.out, 'bench_jpeg.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
