"""Time the torchvision-backed pose models -- ShuffleNetV2 x1, x2 (reference basenetworks.py:36-68) and SqueezeNet 1.1
(basenetworks.py:461-499), each with the CocoKp heads -- on the GPU: the compiled forward alone (CUDA events) and its
time and algorithmic GB/s per op kind, forward + CifCaf decode + fetch through `predictor.Predictor` on planted poses,
and the stock PyTorch forward of the same Shell (fp32, and bf16 channels_last).  Algorithmic bytes are the library's
own count per op (forward_timed: every input once, every output once, the weights once), over the op's event time.

The models are the test mirrors of the reference's modules (tests/torchvision_backbone_models.py) with seeded
from-scratch weights; their heads are calibrated on the backbone features as bench.py does
(network.calibrate_random_heads).  A random net emits no poses, so the decode inside each timed step runs on planted
fields (synth.make_fields, Poisson(4)+1 people per image, one field set per image at the net's field size).

    python tools/bench_shufflenetv2_squeezenet.py --out DIR [--size 641] [--batch 64] [--steps 20] [--warmup 5]

Writes DIR/bench_shufflenetv2_squeezenet.json with the card name, its power limit and max SM clock (nvidia-smi, read
before and after the measurements in the same run)."""
import argparse
import copy
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tools')]
import torchvision_backbone_models as tbm                          # noqa: E402
from bench_mobilenetv2 import card, event_ms, timed                # noqa: E402
from openpifpaf_b200 import constants, network, predictor, synth   # noqa: E402

KINDS = ((0, 'input_conv'), (1, 'gemm'), (2, 'dwconv'), (4, 'maxpool'))    # forward_timed's op kinds


def bench_model(name, size, batch, steps, warmup, dev):
    out = {'model': f'{name} + CocoKp heads'}
    shell = tbm.make_pose_shell(name, seed=0)
    plan = network.plan_from_shell(shell)
    network.calibrate_random_heads(plan, size=min(size, 641), batch=2)
    net = network.CompiledNet(plan, size, size, batch)
    out['gflop_per_image'] = net.flops_per_image / 1e9
    out['ops'] = net.num_ops
    x = torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(1)).to(dev)
    out['compiled_forward_ms'] = event_ms(lambda: net.forward(x), steps, warmup)
    ms, kind, _, nbytes = net.forward_timed(x)
    out['compiled_forward_ms_by_kind'] = {k: float(ms[kind == i].sum()) for i, k in KINDS if (kind == i).any()}
    out['algorithmic_gb_per_s_by_kind'] = {k: float(nbytes[kind == i].sum()) / 1e6 / float(ms[kind == i].sum())
                                           for i, k in KINDS if (kind == i).any()}
    out['algorithmic_gb_per_s'] = float(nbytes.sum()) / 1e6 / float(ms.sum())

    pred = predictor.Predictor(net, constants.COCO_N_KEYPOINTS, constants.COCO_PERSON_SKELETON)
    h, w = net.heads[0]['h'], net.heads[0]['w']
    items = [synth.make_fields('cocokp', h, w, None, 77 * 1000 + b) for b in range(batch)]
    cif = torch.from_numpy(np.stack([it['cif'] for it in items])).to(dev)
    caf = torch.from_numpy(np.stack([it['caf'] for it in items])).to(dev)
    pred.decode_fields_override = (cif, 16, caf, 16)
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
    for label, model, inp in (('fp32', ref32, x), ('bf16_channels_last', ref16, x16)):
        with torch.no_grad():
            out[f'stock_forward_{label}_ms'] = event_ms(lambda: model(inp), steps, warmup)
    del ref32, ref16
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', required=True, help='directory for bench_shufflenetv2_squeezenet.json')
    ap.add_argument('--size', type=int, default=641)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_shufflenetv2_squeezenet.py needs a CUDA device')
    dev = torch.device('cuda', 0)
    torch.backends.cudnn.benchmark = True
    out = {'card': card(), 'size': args.size, 'batch': args.batch, 'steps': args.steps, 'warmup': args.warmup,
           'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32, 'models': {}}
    for name in tbm.NAMES:
        out['models'][name] = bench_model(name, args.size, args.batch, args.steps, args.warmup, dev)
        print(name, json.dumps(out['models'][name]), flush=True)
    out['card_after'] = card()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'bench_shufflenetv2_squeezenet.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
