"""Write tests/golden/opencv_resize.npz: cv2.resize(..., interpolation=cv2.INTER_LINEAR) of seeded uint8 images, so
that the OpenCV rescale can be checked where OpenCV is not installed.  Needs opencv-python.

Each case is (seed, h, w, target_h, target_w); its input is
    numpy.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=numpy.uint8)
and its output is stored as out_<index>.  The file also records cv2.__version__ and the Intel IPP line of
cv2.getBuildInformation(), the build the outputs came from.

    python tools/make_opencv_resize_golden.py
"""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (h, w, target_h, target_w): outputs kept small, so the file stays small
CASES = [
    (37, 53, 61, 45),          # up on both axes: clamped border rows and columns
    (48, 64, 49, 65),          # up by one pixel
    (5, 7, 60, 64),            # large upscale: many rows share the clamped border rows
    (64, 96, 32, 48),          # exactly 2x down on both axes: OpenCV's INTER_AREA fast path
    (64, 95, 32, 40),          # 2x down on rows only
    (60, 90, 25, 45),          # 2x down on columns only
    (120, 90, 41, 57),         # down x up
    (33, 200, 61, 37),         # up x down
    (1, 40, 1, 64),            # 1 x N
    (50, 1, 17, 1),            # N x 1
    (1, 1, 9, 13),             # one pixel -> 9 x 13
    (29, 31, 1, 1),            # -> one pixel
    (1, 57, 3, 9),             # 1 x N -> 3 x 9
    (17, 23, 17, 23),          # unchanged: a copy
    (3024, 4032, 48, 64),      # phone photo, far down
    (4032, 3024, 64, 48),
    (480, 640, 21, 28),
    (97, 131, 100, 129),       # mixed near 1
]


def case_input(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def main():
    import cv2
    ipp = [line.strip() for line in cv2.getBuildInformation().splitlines() if 'Intel IPP:' in line]
    out = {'cv2_version': np.array(cv2.__version__), 'cv2_ipp': np.array(ipp[0] if ipp else 'Intel IPP: NO'),
           'seeds': np.arange(100, 100 + len(CASES), dtype=np.int64),
           'shapes': np.array(CASES, dtype=np.int64)}
    for i, (seed, (h, w, th, tw)) in enumerate(zip(out['seeds'], CASES)):
        out[f'out_{i}'] = cv2.resize(case_input(int(seed), h, w), (tw, th), interpolation=cv2.INTER_LINEAR)
        assert out[f'out_{i}'].shape == (th, tw, 3)
    path = os.path.join(ROOT, 'tests', 'golden', 'opencv_resize.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes; cv2', cv2.__version__, '|', out['cv2_ipp'])


if __name__ == '__main__':
    main()
