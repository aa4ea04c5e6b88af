"""OpenCV-rescale cost: GpuPreprocess(opencv=True) (pifpaf_image_resize_linear_cv_u8, cv2.resize(INTER_LINEAR) +
CenterPad in one launch) against the Pillow path (opencv=False) in the same run, and against cv2.resize on the host
with cv2.setNumThreads(1) and (8).

Inputs: 64 seeded photo-like 640 x 480 images into a 641 x 641 canvas (RescaleAbsolute(641) + CenterPad(641), what
the reference's Predictor does at batch size > 1).  GPU times are CUDA events around the whole call (host images:
including their host-to-device copy; CUDA images: staging and kernel only), median over reps; the kernel alone from
torch.profiler in a separate pass.  The card's name, power limit and SM clocks are read in the same run.  Where
OpenCV is not installed the host rows say so.  Writes DIR/bench_opencv_resize.json and prints it.

    python tools/bench_opencv_resize.py --out DIR [--images 64] [--reps 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_zoom import LONG_EDGE, card, kernel_ms, time_gpu      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--images', type=int, default=64)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import torch
    from openpifpaf_b200 import preprocess as pp
    from openpifpaf_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit('bench_opencv_resize needs a GPU')
    os.makedirs(args.out, exist_ok=True)
    res = {'host': card(), 'canvas': [LONG_EDGE, LONG_EDGE]}
    images = [synth.photo_like_image(480, 640, seed=i) for i in range(args.images)]
    B = len(images)
    tw, th = pp.rescale_target(640, 480, LONG_EDGE)
    left, top, _, _ = pp.center_pad_ltrb(tw, th, LONG_EDGE, LONG_EDGE)
    fills = [(i * 37) % 255 for i in range(B)]
    cuda_images = [torch.from_numpy(im).cuda() for im in images]
    opencv = pp.GpuPreprocess(LONG_EDGE, batched=True, opencv=True)
    pillow = pp.GpuPreprocess(LONG_EDGE, batched=True)
    # the GPU result is OpenCV's (the restatement, and cv2 itself where installed) on the first images
    got = opencv(cuda_images, fill=fills)[0].cpu().numpy()
    try:
        import cv2
    except ImportError:
        cv2 = None
    for i in range(4):
        window = got[i, top:top + th, left:left + tw]
        assert np.array_equal(window, pp.opencv_linear_reference(images[i], tw, th)), i
        if cv2 is not None:
            assert np.array_equal(window, cv2.resize(images[i], (tw, th), interpolation=cv2.INTER_LINEAR)), i
    res.update({'images': B, 'size': [480, 640], 'target': [th, tw],
                'algorithmic_MB_read': sum(im.nbytes for im in images) / 1e6,
                'algorithmic_MB_written': B * LONG_EDGE * LONG_EDGE * 3 / 1e6})
    for label, imgs in (('host_images', images), ('cuda_images', cuda_images)):
        res[f'opencv_{label}'] = time_gpu(lambda: opencv(imgs, fill=fills), args.reps)
        res[f'pillow_{label}'] = time_gpu(lambda: pillow(imgs, fill=fills), args.reps)
    res['opencv_kernel_ms'] = kernel_ms(lambda: opencv(cuda_images, fill=fills), ['k_resize_linear_cv'])
    t0 = time.perf_counter()
    for _ in range(args.reps):
        opencv(cuda_images, fill=fills)
    res['opencv_host_ms_per_call_enqueue'] = (time.perf_counter() - t0) / args.reps * 1e3
    torch.cuda.synchronize()
    if cv2 is None:
        res['cv2'] = 'not installed: host rows not measured'
    else:
        res['cv2'] = cv2.__version__
        for threads in (1, 8):
            cv2.setNumThreads(threads)
            for im in images[:4]:
                cv2.resize(im, (tw, th), interpolation=cv2.INTER_LINEAR)
            t0 = time.perf_counter()
            for _ in range(3):
                for im in images:
                    cv2.resize(im, (tw, th), interpolation=cv2.INTER_LINEAR)
            res[f'cv2_{threads}_threads_ms_per_batch'] = (time.perf_counter() - t0) / 3 * 1e3
    res['host_after'] = card()
    with open(os.path.join(args.out, 'bench_opencv_resize.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
