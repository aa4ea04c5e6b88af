"""CPU: the decoder options of the reference (its CLI flags and C++ statics) through the plain-C oracle, against the
unmodified reference: golden vectors of every option set (tests/golden/options_*.npz), the live reference under every
option set and at CifHr revisions other than the 1.0 of a fresh instance, and the path of each flag from the
reference's CLI into the native decoder's by-value params."""
import hashlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import helpers
from oracle import cifcaf as oc, make_golden

OPTIONS = dict([('default', {})] + make_golden.OPTION_CASES)
# a reused reference instance decodes its n-th call at revision n; 10 000 calls later the buffer wraps to 0
REVISIONS = (2, 4097, 10000, 0)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(autouse=True)
def restore_statics():
    """files that run later assume the default statics, native and reference"""
    yield
    helpers.reset_native_statics()
    if oc.ref_available():
        oc.ref_configure()


def oracle_params(statics, **kw):
    return oc.default_params(**helpers.statics_to_params(statics), **kw)


def golden_id(path):
    return os.path.basename(path)[len('options_'):-len('.npz')]


def test_option_goldens_cover_every_option_and_field():
    want = {make_golden.option_golden_name(o, f) + '.npz'
            for o, _ in make_golden.OPTION_CASES for f in make_golden.OPTION_FIELDS}
    assert {os.path.basename(p) for p in helpers.golden_option_cases()} == want


@pytest.mark.parametrize('path', helpers.golden_option_cases(), ids=golden_id)
def test_oracle_matches_option_golden(path):
    g, f, statics, digest_ok = helpers.load_golden(path)
    assert digest_ok, 'synthetic field generator is not bit-reproducible on this machine'
    option = golden_id(path).split('__')[0]
    assert statics == {k: float(v) for k, v in OPTIONS[option].items()}
    stride = int(g['stride'])
    ann, ids, taps = oc.decode(f['cif'], stride, f['caf'], stride, f['skeleton'], f['n_keypoints'],
                               params=oracle_params(statics), taps=True)
    assert sha(taps['cifhr']) == str(g['cifhr_sha256'])
    assert len(taps['seeds_f']) == int(g['n_seeds'])
    assert sha(taps['seeds_f']) == str(g['seeds_f_sha256'])
    assert sha(taps['seeds_vxys']) == str(g['seeds_vxys_sha256'])
    assert [len(x) for x in taps['fwd']] == list(g['n_fwd'])
    assert [len(x) for x in taps['bwd']] == list(g['n_bwd'])
    if not statics.get('force_complete'):
        assert sha(np.concatenate([x.reshape(-1, 7) for x in taps['fwd']])) == str(g['fwd_sha256'])
        assert sha(np.concatenate([x.reshape(-1, 7) for x in taps['bwd']])) == str(g['bwd_sha256'])
    np.testing.assert_array_equal(ann, g['annotations'])
    np.testing.assert_array_equal(ids, g['ids'])


def _outputs(path):
    g = np.load(path)
    return (str(g['cifhr_sha256']), str(g['seeds_vxys_sha256']) if 'seeds_vxys_sha256' in g else sha(g['seeds_vxys']),
            tuple(g['n_fwd']) + tuple(g['n_bwd']), str(g['fwd_sha256']), g['annotations'].tobytes(), g['ids'].tobytes())


@pytest.mark.parametrize('option', [o for o, _ in make_golden.OPTION_CASES])
def test_every_option_changes_the_reference_output(option):
    """an option golden equal to the default one on every field would test nothing.  Two options are expected to
    change nothing: block_joints has no effect in the reference (cifcaf.cpp:291-295), and no joint of these fields
    scores below half its annotation's best, so keypoint_threshold_rel 0 keeps what 0.5 keeps (kp_rel_1 drops some).
    suppression 0 drops what the default 1e-5 scales below the instance threshold (suppression_1 keeps it)."""
    changed = [_outputs(os.path.join(helpers.GOLDEN_DIR, make_golden.option_golden_name(option, f) + '.npz'))
               != _outputs(os.path.join(helpers.GOLDEN_DIR, f'decoder_{f}.npz'))
               for f in make_golden.OPTION_FIELDS]
    if option in ('block_joints', 'kp_rel_0', 'suppression_0'):
        assert not any(changed)
    else:
        assert any(changed), option


def assert_ref_equals_oracle(ref, orc, lists=True, what=''):
    ra, ri, rt = ref
    oa, oi, ot = orc
    np.testing.assert_array_equal(rt['cifhr'], ot['cifhr'], err_msg=what)
    np.testing.assert_array_equal(rt['seeds_f'], ot['seeds_f'], err_msg=what)
    np.testing.assert_array_equal(rt['seeds_vxys'], ot['seeds_vxys'], err_msg=what)
    if lists:
        for a, b in zip(rt['fwd'] + rt['bwd'], ot['fwd'] + ot['bwd']):
            np.testing.assert_array_equal(a, b, err_msg=what)
    np.testing.assert_array_equal(ra, oa, err_msg=what)
    np.testing.assert_array_equal(ri, oi, err_msg=what)


@pytest.mark.parametrize('option', list(OPTIONS))
def test_oracle_matches_live_reference_under_option(have_reference, option):
    statics = OPTIONS[option]
    have_reference.ref_configure(**statics)
    f = make_golden.live_fields(0)
    ref = have_reference.ref_decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17, taps=True)
    orc = oc.decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17, params=oracle_params(statics), taps=True)
    assert_ref_equals_oracle(ref, orc, lists=not statics.get('force_complete'), what=option)


@pytest.mark.parametrize('option', list(OPTIONS))
def test_oracle_matches_live_reference_at_revisions(have_reference, option):
    """one reference instance decodes at revisions 2, 4097, 10 000 and 0 (ref_decode_revisions); the oracle takes
    the revision as a parameter"""
    statics = OPTIONS[option]
    have_reference.ref_configure(**statics)
    f = make_golden.live_fields(1)
    refs = have_reference.ref_decode_revisions(f['cif'], 16, f['caf'], 16, f['skeleton'], 17, taps=True,
                                               revisions=REVISIONS)
    for r, ref in zip(REVISIONS, refs):
        assert ref[2]['revision'] == float(r)
        orc = oc.decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17,
                        params=oracle_params(statics, cifhr_revision=float(r)), taps=True)
        assert_ref_equals_oracle(ref, orc, lists=not statics.get('force_complete'), what=f'{option} revision {r}')


def test_revisions_change_the_outputs():
    """the revision is not a no-op, so the tests above could see it: above 4096 the map's float32 spacing is 2^-11,
    and at 0 a never-written pixel reads 0 instead of -1"""
    f = make_golden.live_fields(1)
    out = {r: oc.decode(f['cif'], 16, f['caf'], 16, f['skeleton'], 17, taps=True,
                        params=oc.default_params(cifhr_revision=float(r))) for r in (1, 4097, 0)}
    a1, a4097 = out[1][0], out[4097][0]
    assert a1.shape == a4097.shape and len(a1) >= 2
    dv = float(np.abs(a1[..., 0] - a4097[..., 0]).max())
    print(f'max |score(revision 1) - score(revision 4097)| = {dv:.3g}')
    assert dv > 0.0
    hr0 = out[0][2]['cifhr']
    assert (hr0 == 0).any() and not np.array_equal(out[0][2]['seeds_vxys'], out[1][2]['seeds_vxys'])


def test_cifdet_oracle_matches_live_reference_under_options_and_revisions(have_reference):
    f = make_golden.live_det_fields(1)['field']
    for statics in ({}, {'cifhr_threshold': 0.1}, {'cifhr_neighbors': 1}, {'det_seed_threshold': 0.4},
                    {'cifhr_threshold': 0.5, 'cifhr_neighbors': 64, 'det_seed_threshold': 0.05}):
        have_reference.ref_configure(**statics)
        params = {('seed_threshold' if k == 'det_seed_threshold' else k): v for k, v in statics.items()}
        revisions = (1,) + REVISIONS[1:]
        for r, want in zip(revisions, have_reference.ref_decode_det_revisions(f, 16, revisions)):
            got = oc.decode_det(f, 16, params=oc.default_params(cifhr_revision=float(r), **params))
            for a, b in zip(want, got):
                np.testing.assert_array_equal(a, b, err_msg=f'{statics} revision {r}')
            assert len(got[0]) >= 3


def test_ref_configure_resets_every_static(have_reference):
    """ref_configure(**one option) followed by ref_configure() is back at the defaults: the reference's statics are
    process-global"""
    every = {'block_joints': True, 'greedy': True, 'keypoint_threshold': 0.3, 'keypoint_threshold_rel': 0.1,
             'reverse_match': False, 'force_complete': True, 'force_complete_caf_th': 0.2, 'cifhr_neighbors': 3,
             'cifhr_threshold': 0.2, 'cifhr_ablation_skip': True, 'seed_threshold': 0.3, 'seeds_ablation_nms': True,
             'seeds_ablation_no_rescore': True, 'det_seed_threshold': 0.4, 'caf_score_th': 0.4,
             'caf_ablation_no_rescore': True, 'nms_instance_threshold': 0.3, 'nms_keypoint_threshold': 0.25,
             'nms_suppression': 0.5, 'max_detections_before_nms': 777}
    assert set(every) == set(oc.REF_DEFAULTS)
    have_reference.ref_configure(**every)
    got = have_reference.ref_statics()
    assert got == pytest.approx(every) and all(got[k] != v for k, v in oc.REF_DEFAULTS.items())
    have_reference.ref_configure()
    assert have_reference.ref_statics() == pytest.approx(oc.REF_DEFAULTS)
    with pytest.raises(AssertionError):
        have_reference.ref_configure(cif_th=0.1)


def test_native_defaults_equal_reference_defaults(have_reference):
    have_reference.ref_configure()
    from openpifpaf_b200 import decoder
    p = decoder.CifCaf.params()
    for k, v in oc.REF_DEFAULTS.items():
        if hasattr(p, k):
            assert getattr(p, k) == pytest.approx(float(v)), k


# ---- the reference's CLI -> decoder.configure -> sync_statics -> the native decoder's params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='reference package not staged')
def test_reference_cli_reaches_native_params(tmp_path):
    script = textwrap.dedent('''
        import argparse, warnings
        warnings.filterwarnings('ignore')
        import torch
        import openpifpaf
        from openpifpaf_b200 import decoder as N
        dec = {d.__name__: d for d in openpifpaf.DECODERS}
        CifCafB200, CifDetB200 = dec['CifCafB200'], dec['CifDetB200']
        parser = argparse.ArgumentParser()
        openpifpaf.decoder.cli(parser)
        utl = torch.classes.openpifpaf_decoder_utils

        def run(argv):
            openpifpaf.decoder.configure(parser.parse_args(argv))
            CifCafB200.sync_statics()
            CifDetB200.sync_statics()
            p = N.CifCaf.params()
            return {name: getattr(p, name) for name, _ in p._fields_}

        common = ['--cif-th=0.21', '--caf-th=0.17', '--seed-threshold=0.09', '--instance-threshold=0.07',
                  '--greedy', '--cifcaf-block-joints', '--no-reverse-match', '--ablation-cifseeds-nms',
                  '--ablation-cifseeds-no-rescore', '--ablation-caf-no-rescore']
        utl.CifHr.set_neighbors(9)
        utl.NMSKeypoints.set_suppression(0.3)
        torch.classes.openpifpaf_decoder.CifDet.set_max_detections_before_nms(1500)
        p = run(common + ['--keypoint-threshold=0.12', '--keypoint-threshold-rel=0.35'])
        want = dict(cifhr_neighbors=9, cifhr_threshold=0.21, cifhr_ablation_skip=1, seed_threshold=0.09,
                    seeds_ablation_nms=1, seeds_ablation_no_rescore=1, caf_score_th=0.17, caf_ablation_no_rescore=1,
                    block_joints=1, greedy=1, keypoint_threshold=0.09, keypoint_threshold_rel=0.35, reverse_match=1,
                    force_complete=0, force_complete_caf_th=0.001, nms_suppression=0.3, nms_instance_threshold=0.07,
                    nms_keypoint_threshold=0.12, cifhr_revision=1.0)
        # (--no-reverse-match sets the Python class attribute CifCaf.reverse_match, decoder/cifcaf.py:206; the C++
        # static the reference decodes with stays True)
        for k, v in want.items():
            assert p[k] == v, (k, p[k], v)
        # the fields no reference static sets keep the native defaults
        from openpifpaf_b200 import _lib
        d = _lib.default_params()
        for k in set(p) - set(want):
            assert p[k] == getattr(d, k), k
        q = N.CifDet.params()
        assert (q.cifhr_neighbors, q.cifhr_threshold, q.seed_threshold, q.max_detections_before_nms) == \\
            (9, 0.21, 0.09, 1500), (q.cifhr_neighbors, q.cifhr_threshold, q.seed_threshold)
        nms = CifDetB200.nms_params()
        assert nms == dict(iou_threshold=0.5, nms_by_category=True, suppression=0.1, instance_threshold=0.07), nms
        # --force-complete-pose zeroes the keypoint thresholds; --force-complete-caf-th reaches its own param
        p = run(common + ['--force-complete-pose', '--force-complete-caf-th=0.4', '--keypoint-threshold=0.12'])
        assert (p['force_complete'], p['force_complete_caf_th'], p['keypoint_threshold'], p['keypoint_threshold_rel'],
                p['nms_keypoint_threshold']) == (1, 0.4, 0.0, 0.0, 0.0), p
        p = run(['--force-complete-pose', '--force-complete-caf-th=-1'])
        assert (p['force_complete_caf_th'], p['nms_instance_threshold'], p['cifhr_ablation_skip']) == (-1.0, 0.0, 1), p
        print('CLI_OK')
    ''')
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', script], capture_output=True, text=True, env=env, cwd=str(tmp_path),
                       timeout=300)
    assert 'CLI_OK' in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
