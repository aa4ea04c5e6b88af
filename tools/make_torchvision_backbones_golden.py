"""Write tests/golden/torchvision_backbones.npz: the features of the reference's own basenetworks.ShuffleNetV2 (x1, x2)
and SqueezeNet (pretrained off) with the seeded weights of torchvision_backbone_models.make_pose_shell(name, seed=1) on
torchvision_backbone_models.golden_inputs() -- an odd and an even size, the even one where SqueezeNet's ceil-mode pools
add a row and a column.  Keys: input_<size>, <name>_<size>.  Needs the reference sources; torchvision is never asked
for weights.

    python tools/make_torchvision_backbones_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import torchvision_backbone_models as tbm        # noqa: E402


def main():
    inputs = tbm.golden_inputs()
    out = {f'input_{k}': x.numpy() for k, x in inputs.items()}
    for name in tbm.NAMES:
        base = tbm.make_pose_shell(name, seed=1).base_net
        for k, x in inputs.items():
            out[f'{name}_{k}'] = tbm.reference_features(name, x, base).numpy()
    path = os.path.join(ROOT, 'tests', 'golden', 'torchvision_backbones.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, {k: v.shape for k, v in out.items()}, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
