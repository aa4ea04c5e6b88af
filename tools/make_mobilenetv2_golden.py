"""Write tests/golden/mobilenetv2.npz: the features of the reference's own basenetworks.MobileNetV2 (pretrained off)
with the seeded weights of mobilenetv2_models.make_pose_shell(seed=1) on mobilenetv2_models.golden_input().  Needs the
reference sources; torchvision is never asked for weights.

    python tools/make_mobilenetv2_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import mobilenetv2_models as mm        # noqa: E402


def main():
    x = mm.golden_input()
    base = mm.make_pose_shell(seed=1).base_net
    feat = mm.reference_features(x, base).numpy()
    path = os.path.join(ROOT, 'tests', 'golden', 'mobilenetv2.npz')
    np.savez_compressed(path, input=x.numpy(), features=feat)
    print('wrote', path, feat.shape, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
