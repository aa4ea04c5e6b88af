"""Write tests/golden/shufflenetv2k_variants.npz: the features of the reference's own basenetworks.ShuffleNetV2K for
every variant of tests/shufflenetv2k_models.VARIANTS (on the small 'tiny' widths, and conv5-as-stage also on
'tiny_wide', whose conv5 block starts with a branch1), with the seeded weights of
shufflenetv2k_models.make_pose_shell(variant, config, seed=1) on shufflenetv2k_models.golden_input().  Needs the
reference sources.

    python tools/make_shufflenetv2k_variants_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import shufflenetv2k_models as sm        # noqa: E402

# (variant, config) pairs stored; the key is f'{variant}/{config}'
CASES = [(v, 'tiny') for v in sm.VARIANTS] + [('conv5stage', 'tiny_wide')]


def main():
    x = sm.golden_input()
    out = {'input': x.numpy()}
    for v, cfg in CASES:
        base = sm.make_pose_shell(v, cfg, seed=1).base_net
        out[f'{v}/{cfg}'] = sm.reference_features(v, x, base).numpy()
        print(v, cfg, out[f'{v}/{cfg}'].shape)
    path = os.path.join(ROOT, 'tests', 'golden', 'shufflenetv2k_variants.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    torch.set_num_threads(8)
    main()
