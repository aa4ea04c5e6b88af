"""Shared helpers of the test-suite."""
import glob
import os

import numpy as np

from openpifpaf_b200 import synth

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

# parity tolerances of BASELINE.json's north_star
XY_TOL = 1e-4
SCORE_TOL = 1e-5


def golden_cases():
    return sorted(glob.glob(os.path.join(GOLDEN_DIR, 'decoder_*.npz')))


def golden_option_cases():
    """tests/golden/options_*.npz: the reference under non-default decoder options (oracle/make_golden.py OPTION_CASES)"""
    return sorted(glob.glob(os.path.join(GOLDEN_DIR, 'options_*.npz')))


def golden_det_cases():
    return sorted(glob.glob(os.path.join(GOLDEN_DIR, 'cifdet_*.npz')))


def load_golden_det(path):
    import hashlib
    g = np.load(path)
    f = synth.make_det_fields(int(g['n_categories']), int(g['h']), int(g['w']), int(g['n_objects']), int(g['seed']),
                              int(g['n_distractors']))
    digest_ok = hashlib.sha256(np.ascontiguousarray(f['field']).tobytes()).hexdigest() == str(g['field_sha256'])
    return g, f, digest_ok


def load_golden(path):
    g = np.load(path)
    n_people = int(g['n_people'])
    f = synth.make_fields(str(g['workload']), int(g['h']), int(g['w']), None if n_people < 0 else n_people,
                          int(g['seed']), int(g['n_distractors']))
    statics = {str(k): float(v) for k, v in zip(g['statics_keys'], g['statics_vals'])}
    digest_ok = synth.fields_digest(f['cif'], f['caf']) == str(g['fields_sha256'])
    return g, f, statics, digest_ok


FLAG_STATICS = ('greedy', 'force_complete', 'reverse_match', 'block_joints', 'cifhr_ablation_skip', 'seeds_ablation_nms',
                'seeds_ablation_no_rescore', 'caf_ablation_no_rescore', 'cifhr_neighbors')


def statics_to_params(statics):
    """reference static names -> params-struct field values (ints for flags)."""
    out = {}
    for k, v in statics.items():
        out[k] = int(v) if k in FLAG_STATICS else float(v)
    return out


def reset_native_statics():
    """every static of the native decoder classes back to its default (the reference's)"""
    from openpifpaf_b200 import decoder
    for cls in (decoder.CifCaf, decoder.CifHr, decoder.CifSeeds, decoder.CafScored, decoder.NMSKeypoints,
                decoder.CifDetSeeds, decoder.CifDet):
        for name, default in cls.STATICS.items():
            getattr(cls, 'set_' + name)(default)


def assert_annotations_close(got, want, what=''):
    """identical instance count; (v, x, y, s) within the north_star tolerances, instance order included."""
    assert got.shape == want.shape, f'{what}: instance count {got.shape} vs {want.shape}'
    if got.size == 0:
        return
    dv = np.abs(got[..., 0] - want[..., 0]).max()
    dxy = np.abs(got[..., 1:3] - want[..., 1:3]).max()
    ds = np.abs(got[..., 3] - want[..., 3]).max()
    assert dv <= SCORE_TOL, f'{what}: score diff {dv}'
    assert dxy <= XY_TOL, f'{what}: xy diff {dxy}'
    assert ds <= XY_TOL, f'{what}: scale diff {ds}'


def reference_outputs():
    """tests/golden/reference_outputs.npz: what the unmodified reference computed for the cases of oracle/make_golden.py"""
    return np.load(os.path.join(GOLDEN_DIR, 'reference_outputs.npz'))


def assert_taps_match_emulation(net, ops, emu_acts, batch, what=''):
    """After a forward of `net`: every tensor an op of `ops` writes (the heads aside) against the activations of the bf16
    emulation (ops_emulator.run_ops with bf16=True), to 3e-2 of the emulated tensor's largest magnitude."""
    for o in ops:
        if o['kind'] == 'heads':
            continue
        for t_id in sorted({pc[2] for pc in o['pieces']}) if 'pieces' in o else [o['out']]:
            got = net.tap(t_id, batch)
            ref = emu_acts[t_id].numpy()
            scale = max(float(np.abs(ref).max()), 1e-6)
            assert float(np.abs(got - ref).max()) / scale < 3e-2, \
                (what, o['kind'], t_id, o.get('kernel'), o.get('stride'), o.get('dilation'))
