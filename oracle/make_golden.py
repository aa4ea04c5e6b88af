"""Generate tests/golden/*.npz from the UNMODIFIED reference decoder (oracle/_ref).

Run where the reference sources exist (oracle/build_ref.py builds oracle/_ref from them):
    python -m oracle.make_golden
Each fixture stores the generator arguments, the sha256 of the generated float32 fields
(openpifpaf_b200.synth is bit-reproducible, so inputs need not be stored), and the reference's
outputs on a FRESH CifCaf instance: annotations, ids, sorted seeds, per-connection CafScored
counts and a sha256 of the CifHr map.  The smallest case also stores the raw fields.
TEST INFRASTRUCTURE."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openpifpaf_b200 import synth      # noqa: E402
from oracle import cifcaf as oc        # noqa: E402

CASES = [
    # name, workload, h, w, n_people, seed, n_distractors, stride, reference statics
    ('coco11_1p', 'cocokp', 11, 11, 1, 5, 0, 16, {}),
    ('coco11_2p_d3', 'cocokp', 11, 11, 2, 6, 3, 16, {}),
    ('coco41_poisson_s0', 'cocokp', 41, 41, None, 0, 10, 16, {}),
    ('coco41_poisson_s1', 'cocokp', 41, 41, None, 1, 10, 16, {}),
    ('coco31x41_3p', 'cocokp', 31, 41, 3, 12, 0, 16, {}),
    ('coco51_5p_stride8', 'cocokp', 51, 51, 5, 14, 4, 8, {}),
    ('crowd30', 'cocokp', 41, 41, 30, 7, 20, 16, {}),
    ('greedy_4p', 'cocokp', 41, 41, 4, 13, 0, 16, {'greedy': True}),
    ('force_complete_3p', 'cocokp', 41, 41, 3, 11, 5, 16,
     {'force_complete': True, 'keypoint_threshold': 0.0, 'keypoint_threshold_rel': 0.0,
      'nms_keypoint_threshold': 0.0, 'nms_instance_threshold': 0.0}),
    ('wholebody_1p', 'wholebody', 41, 41, 1, 21, 0, 16, {}),
    ('wholebody_4p', 'wholebody', 41, 41, 4, 22, 0, 16, {}),
]


# non-default decoder options (reference CLI flags of decoder/factory.py:52-82 and decoder/cifcaf.py:174-211, or the
# statics of csrc/src/module.cpp), each run on the fields of OPTION_FIELDS: tests/golden/options_<option>__<field>.npz
FORCE_COMPLETE = {'force_complete': True, 'keypoint_threshold': 0.0, 'keypoint_threshold_rel': 0.0,
                  'nms_keypoint_threshold': 0.0, 'nms_instance_threshold': 0.0}     # what --force-complete-pose sets
OPTION_CASES = [
    # name, reference statics
    ('cif_th_0.05', {'cifhr_threshold': 0.05}),                                  # --cif-th
    ('cif_th_0.5', {'cifhr_threshold': 0.5}),
    ('neighbors_1', {'cifhr_neighbors': 1}),                                     # CifHr.neighbors
    ('neighbors_64', {'cifhr_neighbors': 64}),
    ('seed_th_0.01', {'seed_threshold': 0.01, 'keypoint_threshold': 0.01}),     # --seed-threshold (lowers the
    ('seed_th_0.5', {'seed_threshold': 0.5}),                                    # keypoint threshold with it)
    ('caf_th_0.05', {'caf_score_th': 0.05}),                                     # --caf-th
    ('caf_th_0.6', {'caf_score_th': 0.6}),
    ('seeds_nms', {'seeds_ablation_nms': True}),                                 # --ablation-cifseeds-nms
    ('seeds_no_rescore', {'seeds_ablation_no_rescore': True}),                   # --ablation-cifseeds-no-rescore
    ('caf_no_rescore', {'caf_ablation_no_rescore': True}),                       # --ablation-caf-no-rescore
    ('no_rescore_skip', {'seeds_ablation_no_rescore': True, 'caf_ablation_no_rescore': True,
                         'cifhr_ablation_skip': True}),                          # both, which set CifHr.ablation_skip
    ('block_joints', {'block_joints': True}),                                    # --cifcaf-block-joints
    ('kp_rel_0', {'keypoint_threshold_rel': 0.0}),                               # --keypoint-threshold-rel
    ('kp_rel_1', {'keypoint_threshold_rel': 1.0}),
    ('instance_th_0', {'nms_instance_threshold': 0.0}),                          # --instance-threshold
    ('instance_th_0.4', {'nms_instance_threshold': 0.4}),
    ('suppression_0', {'nms_suppression': 0.0}),                                 # NMSKeypoints.suppression
    ('suppression_1', {'nms_suppression': 1.0}),
    ('force_complete', dict(FORCE_COMPLETE, force_complete_caf_th=-1.0)),        # --force-complete-caf-th -1: --caf-th
    ('force_complete_caf_th_0.3', dict(FORCE_COMPLETE, force_complete_caf_th=0.3)),
    ('force_complete_greedy', dict(FORCE_COMPLETE, greedy=True)),
    # evaluation style: --force-complete-pose --seed-threshold 0.01 --cif-th 0.1 --caf-th 0.1 --no-reverse-match
    ('eval', dict(FORCE_COMPLETE, seed_threshold=0.01, cifhr_threshold=0.1, caf_score_th=0.1, reverse_match=False)),
]
OPTION_FIELDS = ['coco41_poisson_s0', 'crowd30', 'wholebody_4p', 'coco51_5p_stride8']       # names of CASES


def option_golden_name(option, field):
    return f'options_{option}__{field}'


DET_CASES = [
    # name, n_categories, h, w, n_objects, seed, n_distractors, stride
    ('det11_3cat_1', 3, 11, 11, 1, 2, 2, 16),
    ('det41_80cat_6', 80, 41, 41, 6, 0, 4, 16),
    ('det21x33_80cat_3', 80, 21, 33, 3, 1, 4, 16),
    ('det51_80cat_150', 80, 51, 51, 150, 4, 10, 8),         # hits max_detections_before_nms = 120
]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def write_decoder_golden(path, workload, h, w, n_people, seed, n_dis, stride, statics, store_fields=False,
                         seed_arrays=True):
    """the reference's outputs under `statics` on a fresh instance, in the layout of tests/golden/decoder_*.npz.
    seed_arrays=False stores the seeds as n_seeds and the sha256 of seeds_f / seeds_vxys (a crowd or WholeBody
    input has thousands of seeds; the option goldens would otherwise take megabytes)."""
    f = synth.make_fields(workload, h, w, n_people, seed, n_dis)
    oc.ref_configure(**statics)
    ann, ids, taps = oc.ref_decode(f['cif'], stride, f['caf'], stride, f['skeleton'], f['n_keypoints'], taps=True)
    if seed_arrays:
        seeds = dict(seeds_f=taps['seeds_f'], seeds_vxys=taps['seeds_vxys'])
    else:
        seeds = dict(n_seeds=len(taps['seeds_f']), seeds_f_sha256=sha(taps['seeds_f']),
                     seeds_vxys_sha256=sha(taps['seeds_vxys']))
    data = dict(
        workload=workload, h=h, w=w, n_people=-1 if n_people is None else n_people, seed=seed,
        n_distractors=n_dis, stride=stride,
        statics_keys=np.array(list(statics.keys()), dtype='U64'),
        statics_vals=np.array([float(v) for v in statics.values()], dtype=np.float64),
        fields_sha256=synth.fields_digest(f['cif'], f['caf']),
        annotations=ann, ids=ids,
        **seeds,
        n_fwd=np.array([len(x) for x in taps['fwd']], dtype=np.int64),
        n_bwd=np.array([len(x) for x in taps['bwd']], dtype=np.int64),
        fwd_sha256=sha(np.concatenate([x.reshape(-1, 7) for x in taps['fwd']])),
        bwd_sha256=sha(np.concatenate([x.reshape(-1, 7) for x in taps['bwd']])),
        cifhr_sha256=sha(taps['cifhr']), cifhr_sum=float(taps['cifhr'].astype(np.float64).sum()),
    )
    if store_fields:
        data['cif'] = f['cif']
        data['caf'] = f['caf']
    np.savez_compressed(path, **data)
    print(os.path.basename(path), 'N =', len(ann), 'seeds =', len(taps['seeds_f']), os.path.getsize(path), 'bytes')


def main():
    out_dir = os.path.join(ROOT, 'tests', 'golden')
    os.makedirs(out_dir, exist_ok=True)
    for name, *args in CASES:
        write_decoder_golden(os.path.join(out_dir, f'decoder_{name}.npz'), *args, store_fields=name == 'coco11_1p')
    oc.ref_configure()
    # CifDet (csrc/src/cifdet.cpp): raw output of a FRESH torch.classes.openpifpaf_decoder.CifDet instance
    for name, n_cat, h, w, n_obj, seed, n_dis, stride in DET_CASES:
        f = synth.make_det_fields(n_cat, h, w, n_obj, seed, n_dis)
        cats, scores, boxes = oc.ref_decode_det(f['field'], stride)
        path = os.path.join(out_dir, f'cifdet_{name}.npz')
        np.savez_compressed(path, n_categories=n_cat, h=h, w=w, n_objects=n_obj, seed=seed, n_distractors=n_dis,
                            stride=stride, field_sha256=sha(f['field']), categories=cats, scores=scores, boxes=boxes)
        print(name, 'N =', len(cats), os.path.getsize(path), 'bytes')


# ---------------------------------------------------------------- what the live-reference tests compare against
def load_reference_modules():
    """basenetworks / heads / headmeta of the reference, loaded by path without running the package __init__
    (which needs the compiled extension and optional dependencies)."""
    import importlib.util
    import types
    from oracle import build_ref
    src = build_ref.REF_PY
    top = types.ModuleType('refpifpaf')
    top.__path__ = [src]
    sys.modules['refpifpaf'] = top
    net_pkg = types.ModuleType('refpifpaf.network')
    net_pkg.__path__ = [os.path.join(src, 'network')]
    sys.modules['refpifpaf.network'] = net_pkg

    def load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod

    top.headmeta = load('refpifpaf.headmeta', os.path.join(src, 'headmeta.py'))
    base = load('refpifpaf.network.basenetworks', os.path.join(src, 'network', 'basenetworks.py'))
    heads = load('refpifpaf.network.heads', os.path.join(src, 'network', 'heads.py'))
    return top.headmeta, base, heads


def reference_constants():
    from oracle import build_ref
    plugins = os.path.join(build_ref.REF_PY, 'plugins')
    ns = {}
    exec(open(os.path.join(plugins, 'coco/constants.py')).read().split('KINEMATIC')[0], ns)
    coco = ns['COCO_PERSON_SKELETON']
    ns = {}
    exec(open(os.path.join(plugins, 'wholebody/constants.py')).read().split('body_kps')[0], ns)
    return coco, ns['WHOLEBODY_SKELETON']


def reference_shufflenet_fields(x):
    """the reference's ShuffleNetV2K + CompositeField4 modules with the weights of net_oracle.make_shell(seed=3)"""
    import torch
    from oracle import net_oracle
    headmeta, base, heads = load_reference_modules()
    ref_base = base.ShuffleNetV2K('shufflenetv2k16', [4, 8, 4], [24, 348, 696, 1392, 1392])
    kps = [str(i) for i in range(17)]
    cif = headmeta.Cif('cif', 'cocokp', keypoints=kps, sigmas=[0.1] * 17)
    caf = headmeta.Caf('caf', 'cocokp', keypoints=kps, sigmas=[0.1] * 17, skeleton=[(1, 2)] * 19)
    ref_heads = [heads.CompositeField4(cif, 1392), heads.CompositeField4(caf, 1392)]
    oracle = net_oracle.make_shell('shufflenetv2k16', seed=3)
    # same parameter names -> load the oracle's (randomised) weights into the reference modules
    ref_base.load_state_dict(oracle.base_net.state_dict())
    for rh, oh in zip(ref_heads, oracle.head_nets):
        rh.load_state_dict(oh.state_dict())
        rh.eval()
    net_oracle.model_defaults(ref_base)
    ref_base.eval()
    with torch.no_grad():
        feat = ref_base(x)
        return [rh(feat) for rh in ref_heads]


def seeded_resnet18():
    """the oracle's resnet18 base with reproducible random weights"""
    import torch
    from oracle import net_oracle
    torch.manual_seed(7)
    oracle = net_oracle.make_base('resnet18')
    oracle.eval()
    return oracle


def reference_resnet18_features(x, oracle):
    """the reference's Resnet module with the weights of `oracle`"""
    import torch
    import torchvision
    _, base, _ = load_reference_modules()
    base.Resnet.pretrained = False
    ref = base.Resnet('resnet18', lambda pretrained: torchvision.models.resnet18(weights=None), 512)
    assert ref.stride == 16
    ref.load_state_dict(oracle.state_dict())
    ref.eval()
    with torch.no_grad():
        return ref(x)


def golden_net_inputs():
    import torch
    g = torch.Generator().manual_seed(20)
    return torch.randn(1, 3, 97, 113, generator=g), torch.randn(1, 3, 161, 161, generator=g)


LIVE_SEEDS = range(4)
LIVE_DET_SEEDS = range(3)


def live_fields(seed):
    return synth.make_fields('cocokp', 21, 27, None, 100 + seed, n_distractors=4)


def live_det_fields(seed):
    return synth.make_det_fields(80, 27, 21, 5 + 20 * seed, 200 + seed, n_distractors=6)


def blend_input():
    rng = np.random.default_rng(0)
    return rng.random((50, 7)).astype(np.float32) * np.array([1, 40, 40, 40, 40, 8, 8], dtype=np.float32)


def initial_annotation_case(decode):
    """a few joints of the first decoded person as initial annotation; `decode` is ref_decode or the oracle's decode"""
    f = synth.make_fields('cocokp', 41, 41, 3, 31)
    base, _ = decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17)
    init = base[:1].copy()
    init[0, 5:] = 0.0          # keep a few joints of the first person, let the decoder regrow the rest
    ids = np.array([42], dtype=np.int64)
    return f, init, ids


def main_reference_outputs():
    """tests/golden/reference_outputs.npz: the reference's side of every comparison the suite otherwise makes live"""
    import torch
    data = {}
    oc.ref_configure()
    for seed in LIVE_SEEDS:
        f = live_fields(seed)
        ann, ids, taps = oc.ref_decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17, taps=True)
        data[f'live{seed}_annotations'] = ann
        data[f'live{seed}_ids'] = ids
        data[f'live{seed}_seeds_vxys'] = taps['seeds_vxys']
        data[f'live{seed}_cifhr_sha256'] = sha(taps['cifhr'])
        data[f'live{seed}_caf_sha256'] = sha(np.concatenate([x.reshape(-1, 7) for x in taps['fwd'] + taps['bwd']]))
    f, init, ids = initial_annotation_case(oc.ref_decode)
    ra, ri = oc.ref_decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17, initial_annotations=init, initial_ids=ids)
    data.update(init_in=init, init_annotations=ra, init_ids=ri)
    oc.load_ref()
    caf = blend_input()
    for only_max in (False, True):
        data[f'blend_{int(only_max)}'] = np.asarray(
            list(torch.ops.openpifpaf_decoder.grow_connection_blend(torch.from_numpy(caf), 20.0, 20.0, 30.0, 1.0, only_max)),
            dtype=np.float64)
    for seed in LIVE_DET_SEEDS:
        cats, scores, boxes = oc.ref_decode_det(live_det_fields(seed)['field'], 16)
        data.update({f'det{seed}_categories': cats, f'det{seed}_scores': scores, f'det{seed}_boxes': boxes})
    coco, wholebody = reference_constants()
    data.update(coco_skeleton=np.asarray(coco, dtype=np.int64), wholebody_skeleton=np.asarray(wholebody, dtype=np.int64))
    x_shuffle, x_resnet = golden_net_inputs()
    cif_f, caf_f = reference_shufflenet_fields(x_shuffle)
    data.update(shufflenet_cif=cif_f.numpy(), shufflenet_caf=caf_f.numpy(),
                resnet18_features=reference_resnet18_features(x_resnet, seeded_resnet18()).numpy())
    path = os.path.join(ROOT, 'tests', 'golden', 'reference_outputs.npz')
    np.savez_compressed(path, **data)
    print('reference_outputs', os.path.getsize(path), 'bytes')


def main_options():
    """tests/golden/options_*.npz: every OPTION_CASES entry on every OPTION_FIELDS input"""
    out_dir = os.path.join(ROOT, 'tests', 'golden')
    cases = {name: args for name, *args in CASES}
    for option, statics in OPTION_CASES:
        for field in OPTION_FIELDS:
            args = cases[field][:-1]
            assert not cases[field][-1]
            write_decoder_golden(os.path.join(out_dir, option_golden_name(option, field) + '.npz'), *args, statics,
                                 seed_arrays=False)
    oc.ref_configure()


if __name__ == '__main__':
    main()
    main_options()
    main_reference_outputs()
