"""Time detection models on the GPU: the compiled forward alone, and forward + CifDet decode + fetch through
`predictor.DetPredictor`, against today's route for a detection model -- a stock PyTorch forward (fp32, and bf16
channels_last), `.cpu()` of the field, then per image `.cuda()` and `decoder.CifDet.decode_batch(nms=True)`.

Models (test mirrors of the reference's modules, tests/det_models.py; from-scratch weights, heads calibrated so that
detections exist):
  resnet18-cocodet        --resnet-input-conv2-stride=2 --resnet-block5-dilation=2, CifDet head with upsample 2
  shufflenetv2k16-cocodet shufflenetv2k16 with the same head (91 categories, upsample 2, as CocoDet builds it)

    python tools/bench_det.py --out DIR [--size 641] [--batch 64] [--steps 10] [--warmup 3]

Writes DIR/bench_det.json with the card name, its power limit and max SM clock (nvidia-smi, same run)."""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import det_models                                     # noqa: E402
from openpifpaf_b200 import decoder, predictor       # noqa: E402
from oracle import net_oracle                         # noqa: E402


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


def models():
    yield 'resnet18-cocodet', det_models.make_variant_shell('cocodet', seed=0)
    yield 'shufflenetv2k16-cocodet', det_models.make_det_shell(net_oracle.make_base('shufflenetv2k16'), 91, 2, seed=0)


def bench(name, shell, size, batch, steps, warmup):
    dev = torch.device('cuda', 0)
    det_models.calibrate_det_head(shell)
    images = torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(1)).pin_memory()
    x = images.to(dev)
    pred = predictor.from_shell(shell, size, size, batch)
    stride = pred.net.heads[0]['stride']
    out = {'model': name, 'size': size, 'batch': batch, 'steps': steps, 'warmup': warmup}
    out['compiled_forward_ms'] = event_ms(lambda: pred.net.forward(x), steps, warmup)

    def compiled_e2e():
        pred.batch_device(x)
        return pred.decoder.fetch()
    out['compiled_forward_decode_fetch_ms'] = timed(compiled_e2e, steps, warmup)
    res = compiled_e2e()
    out['compiled_detections'] = sum(len(c) for c, _, _ in res)
    (field,) = pred.fields_batch(x)
    out['field_shape'] = list(field.shape)
    pred.close()

    dec = decoder.CifDet(91)
    ref32 = shell.to(dev)
    ref16 = copy.deepcopy(ref32).to(dtype=torch.bfloat16, memory_format=torch.channels_last)
    x16 = x.to(dtype=torch.bfloat16, memory_format=torch.channels_last)
    torch.backends.cudnn.benchmark = True

    def today(model, inp):
        with torch.no_grad():
            (f,) = model(inp)
        f = f.float().cpu()                         # decoder/decoder.py:98
        dets = []
        for i in range(f.shape[0]):                 # CifDetB200.__call__ per image: H2D, decode, NMS, fetch
            dets.append(dec.decode_batch(f[i].cuda()[None], stride, nms=True)[0])
        return dets

    for label, model, inp in (('fp32', ref32, x), ('bf16_channels_last', ref16, x16)):
        with torch.no_grad():
            out[f'stock_forward_{label}_ms'] = event_ms(lambda: model(inp), steps, warmup)
        out[f'today_route_{label}_ms'] = timed(lambda: today(model, inp), max(2, steps // 2), 1)
        out[f'today_route_{label}_detections'] = sum(len(c) for c, _, _ in today(model, inp))
    out['images_per_s_compiled'] = batch * 1000.0 / out['compiled_forward_decode_fetch_ms']
    out['images_per_s_today_fp32'] = batch * 1000.0 / out['today_route_fp32_ms']
    out['images_per_s_today_bf16_channels_last'] = batch * 1000.0 / out['today_route_bf16_channels_last_ms']
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', required=True, help='directory for bench_det.json')
    ap.add_argument('--size', type=int, default=641)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_det.py needs a CUDA device')
    # the stock forward runs with PyTorch's defaults (TF32 convolutions allowed), as a user's would
    result = {'card': card(), 'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32, 'models': []}
    for name, shell in models():
        r = bench(name, shell, args.size, args.batch, args.steps, args.warmup)
        print(json.dumps(r), flush=True)
        result['models'].append(r)
        del shell
        torch.cuda.empty_cache()
    result['card_after'] = card()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'bench_det.json'), 'w') as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result['card']))


if __name__ == '__main__':
    main()
