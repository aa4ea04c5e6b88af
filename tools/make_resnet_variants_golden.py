"""Write tests/golden/resnet_variants.npz: the features of the reference's own basenetworks.Resnet for every variant
of tests/det_models.VARIANTS, with the seeded weights of det_models.make_variant_shell(variant, seed=1) on
det_models.golden_variant_input().  Needs the reference sources; torchvision is never asked for weights.

    python tools/make_resnet_variants_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import det_models        # noqa: E402


def main():
    x = det_models.golden_variant_input()
    out = {'input': x.numpy()}
    for v in det_models.VARIANTS:
        base = det_models.make_variant_shell(v, seed=1).base_net
        out[v] = det_models.reference_resnet_features(v, x, base).numpy()
        print(v, out[v].shape)
    path = os.path.join(ROOT, 'tests', 'golden', 'resnet_variants.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    torch.set_num_threads(8)
    main()
