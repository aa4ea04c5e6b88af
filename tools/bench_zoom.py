"""Precise-rescale cost: GpuPreprocess(fast_rescaling=False) (pifpaf_image_zoom_linear_u8, scipy.ndimage.zoom(order=1)
+ CenterPad in one launch) against the Pillow path (fast_rescaling=True) in the same run, and against
scipy.ndimage.zoom on the host, on one core and on all cores.

Inputs: 64 seeded photo-like images into a 641 x 641 canvas (RescaleAbsolute(641) + CenterPad(641), what
--precise-rescaling does at batch size > 1), once all 640 x 480 and once a mixed set of COCO-like sizes.  GPU times
are CUDA events around the whole call (host images: including their host-to-device copy; CUDA images: staging and
kernel only), median over reps; the kernel alone from torch.profiler in a separate pass.  The card's name, power
limit and SM clocks are read in the same run.  Writes DIR/bench_zoom.json and prints it.

    python tools/bench_zoom.py --out DIR [--images 64] [--reps 20]
"""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LONG_EDGE = 641
MIXED = [(640, 480), (640, 427), (480, 640), (427, 640), (500, 375), (612, 612), (640, 360), (375, 500), (640, 512),
         (424, 640), (640, 425), (333, 500)]          # (w, h)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = 'nvidia-smi unavailable'
    return {'gpu (name, power limit, sm clock, max sm clock)': q, 'cpu_count': os.cpu_count()}


def _scipy_zoom(img):
    import scipy.ndimage
    from openpifpaf_b200 import preprocess as pp
    h, w = img.shape[:2]
    tw, th = pp.rescale_target(w, h, LONG_EDGE)
    return scipy.ndimage.zoom(img, (th / h, tw / w, 1), order=1)


def time_gpu(fn, reps):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    st = torch.cuda.current_stream()
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return {'ms_median': float(np.median(times)), 'ms_min': float(np.min(times)), 'ms_max': float(np.max(times))}


def kernel_ms(fn, names):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in names:
            if k in ev.key:
                out[k] = out.get(k, 0.0) + ev.device_time_total / 5 / 1e3
    return out


def run_set(name, images, reps, res):
    import torch
    from openpifpaf_b200 import preprocess as pp
    B = len(images)
    fills = [(i * 37) % 255 for i in range(B)]
    cuda_images = [torch.from_numpy(im).cuda() for im in images]
    precise = pp.GpuPreprocess(LONG_EDGE, batched=True, fast_rescaling=False)
    fast = pp.GpuPreprocess(LONG_EDGE, batched=True, fast_rescaling=True)
    # the GPU result is scipy's, on the first images of the set
    canvas, _ = precise(cuda_images, fill=fills)
    got = canvas.cpu().numpy()
    for i in range(4):
        h, w = images[i].shape[:2]
        tw, th = pp.rescale_target(w, h, LONG_EDGE)
        left, top, _, _ = pp.center_pad_ltrb(tw, th, LONG_EDGE, LONG_EDGE)
        assert np.array_equal(got[i, top:top + th, left:left + tw], _scipy_zoom(images[i])), (name, i)
    src_bytes = sum(im.nbytes for im in images)
    r = {'images': B, 'sizes': sorted({im.shape[:2] for im in images}),
         'algorithmic_MB_read': src_bytes / 1e6, 'algorithmic_MB_written': B * LONG_EDGE * LONG_EDGE * 3 / 1e6}
    for label, imgs in (('host_images', images), ('cuda_images', cuda_images)):
        r[f'precise_{label}'] = time_gpu(lambda: precise(imgs, fill=fills), reps)
        r[f'pillow_{label}'] = time_gpu(lambda: fast(imgs, fill=fills), reps)
    r['precise_kernel_ms'] = kernel_ms(lambda: precise(cuda_images, fill=fills), ['k_zoom_linear'])
    r['pillow_kernels_ms'] = kernel_ms(lambda: fast(cuda_images, fill=fills), ['k_resize_h', 'k_resize_v', 'k_copy_rows',
                                                                             'k_fill_rgb'])
    t0 = time.perf_counter()
    for _ in range(reps):
        precise(cuda_images, fill=fills)
    r['precise_host_ms_per_call_enqueue'] = (time.perf_counter() - t0) / reps * 1e3
    torch.cuda.synchronize()
    # scipy on the host: one core, then one process per core
    t0 = time.perf_counter()
    for im in images[:8]:
        _scipy_zoom(im)
    one = (time.perf_counter() - t0) / 8
    r['scipy_one_core_ms_per_image'] = one * 1e3
    r['scipy_one_core_ms_per_batch'] = one * 1e3 * B
    with mp.get_context('fork').Pool(os.cpu_count()) as pool:
        pool.map(_scipy_zoom, images[:os.cpu_count()])
        t0 = time.perf_counter()
        pool.map(_scipy_zoom, images)
        r['scipy_all_cores_ms_per_batch'] = (time.perf_counter() - t0) * 1e3
    res[name] = r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--images', type=int, default=64)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import scipy
    import torch
    from openpifpaf_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit('bench_zoom needs a GPU')
    os.makedirs(args.out, exist_ok=True)
    res = {'host': card(), 'scipy': scipy.__version__, 'canvas': [LONG_EDGE, LONG_EDGE]}
    flagship = [synth.photo_like_image(480, 640, seed=i) for i in range(args.images)]
    run_set('640x480', flagship, args.reps, res)
    mixed = [synth.photo_like_image(h, w, seed=i) for i, (w, h) in
             zip(range(args.images), [MIXED[i % len(MIXED)] for i in range(args.images)])]
    run_set('mixed', mixed, args.reps, res)
    res['host_after'] = card()
    with open(os.path.join(args.out, 'bench_zoom.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
