"""Synthetic CIF/CAF field workloads ("planted poses") for tests/, smoke() and bench.py.

Random-weight networks emit conf ~ 0.5 everywhere, a degenerate decoder input,
and no pretrained checkpoint can be downloaded here (SURVEY.md 8c gotcha 4).
Decoder inputs are therefore generated: a low-confidence background plus, per
planted person, CIF blobs that vote for each keypoint and CAF cells along each
skeleton edge (recipe of SURVEY.md 8d).

Only +, -, *, / and PCG64 doubles are used (no exp/log), so the generated float32
fields are bit-reproducible on any IEEE machine; golden fixtures can therefore
store (seed, sha256) instead of megabytes of field data.
"""
import hashlib

import numpy as np

from . import constants


def _coco_template():
    # own stick figure, image coordinates (y down), origin at the hip centre, ~10 units tall
    return np.array([
        [0.0, -5.4], [-0.3, -5.7], [0.3, -5.7], [-0.65, -5.5], [0.65, -5.5],
        [-1.5, -4.2], [1.5, -4.2], [-1.9, -2.3], [1.9, -2.2], [-2.0, -0.4], [2.0, -0.3],
        [-1.0, 0.0], [1.0, 0.0], [-1.1, 2.2], [1.1, 2.3], [-1.2, 4.4], [1.2, 4.5],
    ], dtype=np.float64)


def _circle(cx, cy, rx, ry, n, a0=0.0, a1=1.0):
    # n points on an ellipse arc; angles in turns; cos/sin replaced by a rational
    # parametrisation (t -> ((1-t^2)/(1+t^2), 2t/(1+t^2))) to stay exp/trig free.
    pts = []
    for k in range(n):
        u = a0 + (a1 - a0) * (k + 0.5) / n          # turns in [0,1)
        q, r = int(u * 4) % 4, (u * 4) % 1.0         # quadrant + position inside it
        t = r                                        # t in [0,1): quarter arc by rational map
        c, s = (1 - t * t) / (1 + t * t), 2 * t / (1 + t * t)
        for _ in range(q):
            c, s = -s, c
        pts.append([cx + rx * c, cy + ry * s])
    return pts


def _wholebody_template():
    body = _coco_template().tolist()
    feet = [[-1.0, 4.9], [-1.5, 4.9], [-1.25, 4.65], [1.0, 5.0], [1.5, 5.0], [1.25, 4.75]]
    hx, hy = 0.0, -5.45
    face = (
        _circle(hx, hy, 0.85, 0.95, 17, 0.02, 0.48)        # outline 24..40 (lower arc)
        + _circle(hx + 0.35, hy - 0.45, 0.3, 0.12, 5, 0.5, 1.0)   # brow 41..45
        + _circle(hx - 0.35, hy - 0.45, 0.3, 0.12, 5, 0.5, 1.0)   # brow 46..50
        + [[hx, hy - 0.3 + 0.1 * k] for k in range(4)]     # nose bridge 51..54
        + _circle(hx, hy + 0.12, 0.22, 0.08, 5, 0.05, 0.45)       # nostrils 55..59
        + _circle(hx + 0.33, hy - 0.25, 0.14, 0.07, 6)            # eye 60..65
        + _circle(hx - 0.33, hy - 0.25, 0.14, 0.07, 6)            # eye 66..71
        + _circle(hx, hy + 0.5, 0.34, 0.16, 12)                   # outer lip 72..83
        + _circle(hx, hy + 0.5, 0.2, 0.07, 8)                     # inner lip 84..91
    )

    def hand(wx, wy, sign):
        pts = [[wx, wy + 0.15]]
        for fngr in range(5):
            dx = sign * (-0.3 + 0.15 * fngr)
            for seg in range(4):
                pts.append([wx + dx * (1 + 0.35 * seg), wy + 0.3 + 0.17 * seg + 0.02 * fngr])
        return pts

    lh = hand(-2.0, -0.4, -1.0)
    rh = hand(2.0, -0.3, 1.0)
    out = np.array(body + feet + face + lh + rh, dtype=np.float64)
    assert out.shape == (133, 2), out.shape
    return out


WORKLOADS = {
    # name: (n_keypoints, skeleton (1-based), template, person scale range, joint scale factor)
    'cocokp': (17, constants.COCO_PERSON_SKELETON, _coco_template, (0.6, 1.1), 0.5),
    'wholebody': (133, None, _wholebody_template, (2.2, 3.0), 0.15),
}


def skeleton_for(workload):
    if workload == 'wholebody':
        return constants.wholebody_skeleton()
    return WORKLOADS[workload][1]


def _poisson(rng, lam):
    # Knuth, on PCG64 doubles only (np.random's poisson may change across versions)
    limit, k, prod = 1.0, 0, rng.random()
    # exp(-lam) via repeated halving-free product: compare prod against e^-lam computed
    # by its Taylor series in exact order (deterministic IEEE arithmetic)
    e = 1.0
    term = 1.0
    for n in range(1, 60):
        term = term * lam / n
        e += term
    limit = 1.0 / e
    while prod > limit:
        k += 1
        prod *= rng.random()
    return k


def make_fields(workload='cocokp', h=41, w=41, n_people=None, seed=0,
                n_distractors=0, people_lambda=4.0, skeleton=None, poses=None):
    """One image worth of fields.

    Returns dict(cif [F,5,h,w] f32, caf [C,8,h,w] f32, skeleton [C,2] int64 0-based,
    n_keypoints, n_planted, keypoints [n_planted,K,2] in field units).
    n_people=None draws Poisson(people_lambda)+1 (COCO-like).  skeleton: optional 1-based connection list replacing the
    workload's own (e.g. the sparse + dense COCO connections of CifCafDense).  poses: optional list of
    (keypoints [K,2] in field units, person scale) to plant instead of randomly placed ones (tracking sequences)."""
    K, _, template_fn, (smin, smax), joint_scale = WORKLOADS[workload]
    skeleton1 = np.asarray(skeleton_for(workload) if skeleton is None else skeleton, dtype=np.int64)
    C = skeleton1.shape[0]
    rng = np.random.Generator(np.random.PCG64(seed))
    template = template_fn()
    if poses is not None:
        n_people = len(poses)
    if n_people is None:
        n_people = _poisson(rng, people_lambda) + 1

    cif = np.zeros((K, 5, h, w), dtype=np.float64)
    caf = np.zeros((C, 8, h, w), dtype=np.float64)
    ii, jj = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    cif[:, 1] = rng.random((K, h, w)) * 0.05
    cif[:, 2] = ii
    cif[:, 3] = jj
    cif[:, 4] = 1.0
    caf[:, 1] = rng.random((C, h, w)) * 0.05
    caf[:, 2] = ii
    caf[:, 3] = jj
    caf[:, 4] = ii
    caf[:, 5] = jj
    caf[:, 6] = 1.0
    caf[:, 7] = 1.0

    tmin, tmax = template.min(axis=0), template.max(axis=0)
    planted = []
    for person in range(n_people):
        if poses is not None:
            kps, ps = np.asarray(poses[person][0], dtype=np.float64), float(poses[person][1])
        else:
            ps = smin + (smax - smin) * rng.random()
            ext = (tmax - tmin) * ps
            # keep the whole pose inside the field with a 1-cell margin where possible
            ox = 1.0 + rng.random() * max(w - 3.0 - ext[0], 0.0) - tmin[0] * ps
            oy = 1.0 + rng.random() * max(h - 3.0 - ext[1], 0.0) - tmin[1] * ps
            kps = template * ps + np.array([ox, oy])
            kps = kps + (rng.random(kps.shape) - 0.5) * 0.2          # per-joint jitter
        planted.append(kps)
        sc = joint_scale * ps
        for k in range(K):
            x, y = kps[k]
            i0, i1 = max(int(np.floor(x - 3)), 0), min(int(np.ceil(x + 3)), w - 1)
            j0, j1 = max(int(np.floor(y - 3)), 0), min(int(np.ceil(y + 3)), h - 1)
            for j in range(j0, j1 + 1):
                for i in range(i0, i1 + 1):
                    d2 = (i - x) * (i - x) + (j - y) * (j - y)
                    if d2 > 6.5:
                        continue
                    g = (1.0 - d2 / 20.0)
                    conf = 0.95 * g * g - 0.01 * rng.random()
                    if conf <= cif[k, 1, j, i]:
                        continue
                    cif[k, 1, j, i] = conf
                    cif[k, 2, j, i] = x + 0.002 * (i - x)
                    cif[k, 3, j, i] = y + 0.002 * (j - y)
                    cif[k, 4, j, i] = sc
        for c in range(C):
            a, b = skeleton1[c] - 1
            xa, ya = kps[a]
            xb, yb = kps[b]
            length = abs(xb - xa) + abs(yb - ya)
            n_steps = int(length / 0.5) + 1
            for st in range(n_steps + 1):
                t = st / n_steps
                px, py = xa + t * (xb - xa), ya + t * (yb - ya)
                for dj in (0, 1):
                    for di in (0, 1):
                        i, j = int(np.floor(px)) + di, int(np.floor(py)) + dj
                        if i < 0 or i >= w or j < 0 or j >= h:
                            continue
                        conf = 0.9 - 0.02 * rng.random()
                        if conf <= caf[c, 1, j, i]:
                            continue
                        caf[c, 1, j, i] = conf
                        caf[c, 2, j, i] = xa + 0.002 * (i - px)
                        caf[c, 3, j, i] = ya + 0.002 * (j - py)
                        caf[c, 4, j, i] = xb + 0.002 * (i - px)
                        caf[c, 5, j, i] = yb + 0.002 * (j - py)
                        caf[c, 6, j, i] = sc
                        caf[c, 7, j, i] = sc

    # distractors: isolated CIF blobs without CAF support (-> one-joint annotations, dropped by NMS)
    for _ in range(n_distractors):
        k = int(rng.random() * K) % K
        x, y = rng.random() * (w - 1), rng.random() * (h - 1)
        peak = 0.5 + 0.45 * rng.random()
        sc = 0.3 + 0.5 * rng.random()
        for j in range(max(int(y) - 2, 0), min(int(y) + 3, h - 1) + 1):
            for i in range(max(int(x) - 2, 0), min(int(x) + 3, w - 1) + 1):
                d2 = (i - x) * (i - x) + (j - y) * (j - y)
                if d2 > 6.5:
                    continue
                g = (1.0 - d2 / 20.0)
                conf = peak * g * g - 0.01 * rng.random()
                if conf <= cif[k, 1, j, i]:
                    continue
                cif[k, 1, j, i] = conf
                cif[k, 2, j, i] = x + 0.01 * (i - x)
                cif[k, 3, j, i] = y + 0.01 * (j - y)
                cif[k, 4, j, i] = sc

    return {
        'cif': cif.astype(np.float32), 'caf': caf.astype(np.float32),
        'skeleton': (skeleton1 - 1).astype(np.int64), 'n_keypoints': K,
        'n_planted': n_people,
        'keypoints': np.asarray(planted, dtype=np.float64).reshape(n_people, K, 2),
    }


def make_tracking_sequence(h=33, w=41, n_people=4, n_frames=4, seed=0, step=0.45):
    """Fields of a COCO-17 tracking model (TSingleImageCif, TSingleImageCaf, Tcaf heads; decoder/tracking_pose.py) for
    `n_frames` consecutive frames of `n_people` planted people drifting by up to `step` cells per frame.

    Returns a list of dict(cif [17,5,h,w], caf [19,8,h,w], tcaf [17,8,h,w], keypoints [n,17,2]); the Tcaf field of
    joint k connects the joint in THIS frame (x1, y1) with the same joint in the PREVIOUS frame (x2, y2), headmeta.py
    Tcaf.skeleton; frame 0 has background only."""
    K, _, template_fn, (smin, smax), joint_scale = WORKLOADS['cocokp']
    rng = np.random.Generator(np.random.PCG64(seed + 77))
    first = make_fields('cocokp', h, w, n_people, seed)
    scales = []
    for kps in first['keypoints']:
        ext = kps.max(axis=0) - kps.min(axis=0)
        t = template_fn()
        scales.append(float(ext[1] / (t[:, 1].max() - t[:, 1].min())))
    poses = [np.asarray(k, dtype=np.float64) for k in first['keypoints']]
    velocity = [(rng.random(2) - 0.5) * 2.0 * step for _ in poses]
    frames, prev = [], None
    for t in range(n_frames):
        f = make_fields('cocokp', h, w, seed=seed * 100 + t, poses=[(p, s) for p, s in zip(poses, scales)])
        ii, jj = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
        tcaf = np.zeros((K, 8, h, w), dtype=np.float64)
        tcaf[:, 1] = rng.random((K, h, w)) * 0.05
        tcaf[:, 2] = ii; tcaf[:, 3] = jj; tcaf[:, 4] = ii; tcaf[:, 5] = jj
        tcaf[:, 6] = 1.0; tcaf[:, 7] = 1.0
        if prev is not None:
            for p_now, p_old, ps in zip(poses, prev, scales):
                sc = joint_scale * ps
                for k in range(K):
                    xa, ya = p_now[k]
                    xb, yb = p_old[k]
                    for dj in (-1, 0, 1):
                        for di in (-1, 0, 1):
                            i, j = int(np.floor(xa)) + di, int(np.floor(ya)) + dj
                            if i < 0 or i >= w or j < 0 or j >= h:
                                continue
                            conf = 0.9 - 0.02 * rng.random()
                            if conf <= tcaf[k, 1, j, i]:
                                continue
                            tcaf[k, 1, j, i] = conf
                            tcaf[k, 2, j, i] = xa + 0.002 * (i - xa)
                            tcaf[k, 3, j, i] = ya + 0.002 * (j - ya)
                            tcaf[k, 4, j, i] = xb + 0.002 * (i - xa)
                            tcaf[k, 5, j, i] = yb + 0.002 * (j - ya)
                            tcaf[k, 6, j, i] = sc
                            tcaf[k, 7, j, i] = sc
        frames.append({'cif': f['cif'], 'caf': f['caf'], 'tcaf': tcaf.astype(np.float32),
                       'keypoints': np.asarray(poses).copy()})
        prev = [p.copy() for p in poses]
        poses = [p + v + (rng.random(p.shape) - 0.5) * 0.05 for p, v in zip(poses, velocity)]
    return frames


def make_batch(workload='cocokp', batch=8, h=41, w=41, n_people=None, seed=0, n_distractors=0):
    """Batch of fields: cif [B,F,5,h,w], caf [B,C,8,h,w] (float32 numpy)."""
    items = [make_fields(workload, h, w, n_people, seed * 1000 + b, n_distractors) for b in range(batch)]
    return {
        'cif': np.stack([it['cif'] for it in items]), 'caf': np.stack([it['caf'] for it in items]),
        'skeleton': items[0]['skeleton'], 'n_keypoints': items[0]['n_keypoints'],
        'n_planted': [it['n_planted'] for it in items],
    }


def make_det_fields(n_categories=80, h=41, w=41, n_objects=6, seed=0, n_distractors=4, n_overlapping=0):
    """One image worth of CifDet fields ("planted boxes"): [F,6,h,w] f32 -- intensity(unused), confidence, x, y
    (cell index added, like the eval head), w, h in field units (headmeta.py:117-134; csrc/src/cif_hr.cpp:124-150
    reads components 1..5).  Per planted object of category f, every cell within ~2.5 cells of its centre votes for
    the centre with a bump-shaped confidence; a few cells carry a NEGATIVE width (skipped by `w < min_scale`), and
    near-duplicate objects of the same category test the occupancy suppression.  Distractors are weak blobs (some
    between the CifHr threshold 0.3 and the seed threshold 0.2).
    Returns dict(field, n_planted, boxes [n,5] (category 1-based, cx, cy, w, h))."""
    rng = np.random.Generator(np.random.PCG64(seed))
    F = n_categories
    field = np.zeros((F, 6, h, w), dtype=np.float64)
    ii, jj = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    field[:, 1] = rng.random((F, h, w)) * 0.05
    field[:, 2] = ii
    field[:, 3] = jj
    field[:, 4] = 1.0
    field[:, 5] = 1.0
    planted = []

    def plant(f, x, y, bw, bh, peak, radius2=6.5):
        for j in range(max(int(y) - 3, 0), min(int(y) + 4, h - 1) + 1):
            for i in range(max(int(x) - 3, 0), min(int(x) + 4, w - 1) + 1):
                d2 = (i - x) * (i - x) + (j - y) * (j - y)
                if d2 > radius2:
                    continue
                g = (1.0 - d2 / 20.0)
                conf = peak * g * g - 0.01 * rng.random()
                if conf <= field[f, 1, j, i]:
                    continue
                field[f, 1, j, i] = conf
                field[f, 2, j, i] = x + 0.002 * (i - x)
                field[f, 3, j, i] = y + 0.002 * (j - y)
                field[f, 4, j, i] = bw * (1.0 + 0.01 * (rng.random() - 0.5))
                field[f, 5, j, i] = bh * (1.0 + 0.01 * (rng.random() - 0.5))

    for n in range(n_objects):
        f = int(rng.random() * F) % F
        bw, bh = 1.5 + rng.random() * 0.3 * w, 1.5 + rng.random() * 0.3 * h
        x = 1.0 + rng.random() * (w - 3.0)
        y = 1.0 + rng.random() * (h - 3.0)
        plant(f, x, y, bw, bh, 0.95)
        planted.append([f + 1, x, y, bw, bh])
        if n % 3 == 2:        # a near duplicate of the same category, half a cell away: suppressed by the occupancy
            plant(f, x + 0.5, y + 0.25, bw * 1.1, bh * 0.9, 0.7, radius2=2.5)
    for _ in range(n_distractors):
        f = int(rng.random() * F) % F
        x, y = rng.random() * (w - 1), rng.random() * (h - 1)
        plant(f, x, y, 1.0 + 3.0 * rng.random(), 1.0 + 3.0 * rng.random(), 0.22 + 0.3 * rng.random(), radius2=2.5)
    # pairs of large same-category boxes 1.5 cells apart: far enough to escape each other's occupancy mark, close
    # enough for IoU ~ 0.6 -- work for the NMS of decoder/cifdet.py:55-64 (drawn after everything above, so the
    # fields of n_overlapping == 0 are unchanged)
    for _ in range(n_overlapping):
        f = int(rng.random() * F) % F
        bw, bh = 8.0 + 2.0 * rng.random(), 8.0 + 2.0 * rng.random()
        x = 2.0 + rng.random() * (w - 6.0)
        y = 2.0 + rng.random() * (h - 5.0)
        plant(f, x, y, bw, bh, 0.9)
        plant(f, x + 1.5, y + 0.5, bw * 1.03, bh * 0.97, 0.75, radius2=2.5)
    # a few cells with a negative width / height (never contribute to the hi-res map, still become seeds)
    for _ in range(3 if n_overlapping == 0 else 0):
        f = int(rng.random() * F) % F
        i, j = int(rng.random() * w) % w, int(rng.random() * h) % h
        field[f, 1, j, i] = 0.6 + 0.2 * rng.random()
        field[f, 4, j, i] = -0.5
    return {'field': field.astype(np.float32), 'n_planted': n_objects,
            'boxes': np.asarray(planted, dtype=np.float64).reshape(n_objects, 5)}


def fields_digest(cif, caf):
    m = hashlib.sha256()
    m.update(np.ascontiguousarray(cif, dtype=np.float32).tobytes())
    m.update(np.ascontiguousarray(caf, dtype=np.float32).tobytes())
    return m.hexdigest()


def photo_like_image(h, w, seed=0):
    """uint8 [h, w, 3] with the statistics JPEG encoders meet in photographs: smooth colour fields, oriented texture
    and sensor-like noise (seeded; the input of the JPEG decode tests and tools/bench_jpeg.py)"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.zeros((h, w, 3))
    for c in range(3):
        for _ in range(3):                                  # smooth fields
            fx, fy = rng.uniform(0.2, 3.0, 2) * 2 * np.pi / max(h, w)
            img[..., c] += rng.uniform(20, 60) * np.sin(fx * x + fy * y + rng.uniform(0, 2 * np.pi))
        img[..., c] += rng.uniform(60, 190)
    a = rng.uniform(0, np.pi)                               # texture
    img += rng.uniform(5, 25) * np.sin((np.cos(a) * x + np.sin(a) * y) * rng.uniform(0.3, 1.2))[..., None]
    img += rng.normal(0, rng.uniform(2, 10), img.shape)     # noise
    return np.clip(img, 0, 255).astype(np.uint8)
