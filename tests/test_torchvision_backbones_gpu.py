"""GPU: ShuffleNetV2 x1 / x2 and SqueezeNet 1.1 in the compiled forward.  The ceil-mode k_maxpool bit for bit against
torch.max_pool2d(ceil_mode=True) on the same bf16 tensor; a Fire module's expand pair writing the two column windows of
one tensor (and nothing outside them) against float64; each seeded family op by op against the float64 reference of what
the GPU fed each op and against fp32 PyTorch; a net compiled at one capacity run at sizes of every residue mod 16
(even sizes included, where the ceil rule adds a row or a column) bit for bit against a net compiled at each size;
Predictor / DetPredictor from the Shell against the decoders on the compiled fields; and the reference's own Predictor
with --basenet shufflenetv2x1 and squeezenet through the plugin.  Sentinels, bounds and column windows are those of
tests/test_kernels_gpu.py."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import det_models
import input_size_models as ism
import kernel_refs as kr
import mobilenetv2_models as mm
import torchvision_backbone_models as tbm
from openpifpaf_b200 import _lib, decoder, network, predictor
from test_input_size_gpu import assert_same, run
from test_kernels_gpu import Case, Check, pad8, pad16, ptr, record
from test_torchvision_backbones import field_tol

pytestmark = pytest.mark.gpu

LAYOUTS = [('shufflenetv2x1', 'bins'), ('shufflenetv2x1', 'shuffle'), ('shufflenetv2x2', 'bins'),
           ('squeezenet', None)]


# ---------------------------------------------------------------------------------------------------- max pool
# (H, W, channels, stride, in_off, out_off, batch, max_batch)
POOL_CASES = [
    (1, 1, 8, 2, 0, 0, 1, 2),
    (2, 2, 16, 2, 0, 8, 2, 3),            # the ceil rule's window reaches two taps past the image
    (4, 6, 64, 2, 8, 0, 2, 2),
    (320, 320, 64, 2, 0, 0, 2, 2),        # the stem output of a 640 px image: 161, not 160
    (161, 161, 64, 2, 0, 0, 2, 2),        # the stem output of a 321 px image (odd: the ceil rule does not fire)
    (160, 81, 128, 2, 16, 0, 2, 3),
    (40, 41, 256, 2, 0, 16, 1, 2),
    (17, 16, 20, 1, 0, 0, 2, 3),          # stride 1: ceil and floor agree
    (16, 17, 64, 1, 8, 8, 2, 2),
]


def pool_id(c):
    return 'H%dW%d-C%d-s%d-in%d-out%d-B%dof%d' % c


@pytest.mark.parametrize('c', POOL_CASES, ids=pool_id)
def test_ceil_mode_maxpool_equals_torch_bitwise(c):
    H, W, C, s, in_off, out_off, batch, mb = c
    Ho, Wo = network.conv_out_hw(H, W, 3, s, 1, ceil_mode=True)
    case = Case(mb, [(H, W, pad16(in_off + C + 8)), (Ho, Wo, pad16(out_off + pad8(C) + 8))], inputs={0})

    def emit(L, net):
        _lib.check(L.pifpaf_net_maxpool_ceil(net, 0, in_off, C, s, 1, out_off, 1))

    def pool(cols):
        x = torch.from_numpy(case.data[0][:batch, ..., cols]).cuda().to(torch.bfloat16).permute(0, 3, 1, 2)
        return torch.max_pool2d(x, 3, s, 1, ceil_mode=True).permute(0, 2, 3, 1).float().cpu().numpy()

    want = pool(slice(in_off, in_off + C))
    assert want.shape[1:3] == (Ho, Wo)
    taps, _ = case.run(emit, batch)
    chk = Check('maxpool ceil', batch)
    chk.own(1, out_off, out_off + pad8(C))
    chk.exact(1, out_off, want)
    if pad8(C) > C:         # padding columns of the input window hold random values: the pool passes them through
        chk.exact(1, out_off + C, pool(slice(in_off + C, in_off + pad8(C))))
    assert chk.verify(taps, pool_id(c)) == 0.0


def test_maxpool_ceil_entry_checks_its_arguments():
    """ceil_mode 0 is pifpaf_net_maxpool; another ceil_mode value, and a table at the floor size, are refused"""
    H, W, C = 20, 22, 32
    case = Case(1, [(H, W, C), (11, 12, C), (10, 11, C)], inputs={0})

    def emit(L, net):
        assert L.pifpaf_net_maxpool_ceil(net, 0, 0, C, 2, 1, 0, 2) == _lib.E_BADARG
        assert L.pifpaf_net_maxpool_ceil(net, 0, 0, C, 2, 1, 0, 0) == _lib.E_BADARG      # 11 x 12 is the ceil size
        assert L.pifpaf_net_maxpool_ceil(net, 0, 0, C, 2, 2, 0, 1) == _lib.E_BADARG      # 10 x 11 is the floor size
        _lib.check(L.pifpaf_net_maxpool_ceil(net, 0, 0, C, 2, 2, 0, 0))
        _lib.check(L.pifpaf_net_maxpool_ceil(net, 0, 0, C, 2, 1, 0, 1))
        assert L.pifpaf_net_num_ops(net) == 2

    taps, _ = case.run(emit, 1)
    x = torch.from_numpy(case.data[0][:1]).permute(0, 3, 1, 2)
    np.testing.assert_array_equal(taps[2], torch.max_pool2d(x, 3, 2, 1).permute(0, 2, 3, 1).numpy())
    np.testing.assert_array_equal(taps[1], torch.max_pool2d(x, 3, 2, 1, ceil_mode=True).permute(0, 2, 3, 1).numpy())


# ---------------------------------------------------------------------------------------------------- Fire expand pair
# (H, W, squeeze channels, expand1x1, expand3x3, batch, max_batch)
FIRE_CASES = [
    (161, 161, 16, 64, 64, 2, 2),         # fire2 of a 641 px image
    (41, 41, 64, 256, 256, 2, 3),         # fire9
    (13, 7, 48, 192, 192, 1, 2),
    (9, 11, 32, 32, 40, 2, 2),            # unequal halves, the second one 40 channels from column 32
]


def fire_id(c):
    return 'H%dW%d-sq%d-e%d-e%d-B%dof%d' % c


@pytest.mark.parametrize('c', FIRE_CASES, ids=fire_id)
def test_fire_expand_pair_writes_its_two_column_windows(c):
    H, W, S, E1, E3, batch, mb = c
    width = pad16(E1 + E3) + 16               # 16 more columns than the pair owns: they must keep the sentinel
    case = Case(mb, [(H, W, pad16(S)), (H, W, width)], inputs={0})
    rng = np.random.default_rng(E1 + E3)
    w1 = kr.random_bf16(rng, (E1, S, 1, 1), 1 / np.sqrt(S))
    w3 = kr.random_bf16(rng, (E3, S, 3, 3), 1 / np.sqrt(9 * S))
    b1 = rng.uniform(-0.5, 0.5, E1).astype(np.float32)
    b3 = rng.uniform(-0.5, 0.5, E3).astype(np.float32)

    def emit(L, net):
        _lib.check(L.pifpaf_net_conv(net, 0, 0, S, 1, 1, 0, E1, ptr(w1), ptr(b1), 1, 1, 0, -1, 0))
        _lib.check(L.pifpaf_net_conv(net, 0, 0, S, 3, 1, 1, E3, ptr(w3), ptr(b3), 1, 1, E1, -1, 0))

    x = case.data[0][:batch, ..., :S]
    chk = Check('fire expand', batch)
    chk.own(1, 0, E1 + pad8(E3))
    for c0, w, b, k in ((0, w1, b1, 1), (E1, w3, b3, 3)):
        ref, mag = kr.epilogue(*kr.conv_ref(x, w, b, 1, (k - 1) // 2), 1)
        chk.compare(1, c0, ref, kr.bf16_bound(ref, mag, S * k * k))
    for impl in (0, 1):
        taps, _ = case.run(emit, batch, impl=impl)
        print(fire_id(c), impl, '%.3f' % chk.verify(taps, f'{fire_id(c)} impl {impl}'))
        assert (taps[1][..., E1 + pad8(E3):] == kr.SENTINEL).all()


# ---------------------------------------------------------------------------------------------------- networks
def teacher_forced(net, ops, images, label):
    """check_ops_teacher_forced (tests/test_kernels_gpu.py), the ceil-mode pools compared at every output pixel
    (kernel_refs.maxpool_ref's whole-tensor form has the floor size)"""
    B = images.shape[0]
    fields = [t.clone() for t in net.forward(torch.from_numpy(images).cuda())]
    torch.cuda.synchronize()
    taps = {t: net.tap(t, B) for t in range(len(net.tensor_shapes))}
    heads = [t.cpu().numpy() for t in fields]
    worst = {}
    for i, o in enumerate(ops):
        pos = None
        if o.get('ceil_mode'):
            ho, wo, _ = net.tensor_shapes[o['out']]
            pos = np.stack(np.meshgrid(np.arange(B), np.arange(ho), np.arange(wo), indexing='ij'), -1).reshape(-1, 3)
        kind, r = kr.op_ref(o, taps, heads, images, B, positions=pos)
        worst[kind] = max(worst.get(kind, 0.0), r)
        record(f'{kind} ({label})', r, f'op {i}')
    return worst, fields


@pytest.mark.parametrize('H,W', [(641, 641), (353, 481), (352, 480)])
@pytest.mark.parametrize('name,layout', LAYOUTS)
def test_network_teacher_forced(name, layout, H, W):
    shell = tbm.make_pose_shell(name, seed=4)
    plan = network.plan_from_shell(shell)
    _, ops, _ = network.build_ops(plan, H, W, layout=layout)
    net = network.CompiledNet(plan, H, W, 2, layout=layout)
    images = np.random.default_rng(9).standard_normal((2, 3, H, W)).astype(np.float32)
    worst, _ = teacher_forced(net, ops, images, name)
    print(name, layout, H, W, {k: round(v, 3) for k, v in worst.items()})
    assert all(v <= 1.0 for v in worst.values()), worst
    x = torch.from_numpy(images).cuda()
    _, kind, _, _ = net.forward_timed(x)
    # ShuffleNetV2: no fused launch (kind 3) -- the 3x3 depthwise convs run alone; SqueezeNet: 3 max pools (kind 4)
    want = [0, 1, 2] if name != 'squeezenet' else [0, 1, 4]
    assert sorted(set(kind.tolist())) == want
    net.close()


@pytest.mark.parametrize('H,W,B', [(641, 641, 64), (353, 481, 8)])
@pytest.mark.parametrize('name', tbm.NAMES)
def test_network_against_fp32(name, H, W, B):
    shell = tbm.make_pose_shell(name, seed=4)
    net = network.CompiledNet(network.plan_from_shell(shell), H, W, B)
    x = torch.from_numpy(np.random.default_rng(10).standard_normal((B, 3, H, W)).astype(np.float32)).cuda()
    got = [t.clone() for t in net.forward(x)]
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        want = shell.cuda()(x)
    assert got[0].shape[-2:] == ((H - 1) // 16 + 1, (W - 1) // 16 + 1)
    for g, wt in zip(got, want):
        assert g.shape == wt.shape
        err = (g - wt).abs()
        print(name, H, W, float(err.max() / wt.std()), float(err.mean() / wt.std()))
        assert float(err.max()) < field_tol(name) * float(wt.std()) + 1e-3
        assert float(err.mean()) < 1e-2 * float(wt.std())
    net.close()


CAP = (161, 193)            # tests/test_input_size_gpu.py


@pytest.mark.parametrize('name,layout', LAYOUTS)
def test_each_size_equals_a_net_compiled_at_it(name, layout):
    plan = network.plan_from_shell(tbm.make_pose_shell(name, seed=9))
    net = network.CompiledNet(plan, *CAP, 3, layout=layout)
    sizes = ism.sizes(*CAP) + [(15, 13), (160, 192)]
    assert any(h % 2 == 0 for h, _ in sizes) and any(w % 2 == 0 for _, w in sizes)
    for i, (h, w) in enumerate(sizes):
        ref = network.CompiledNet(plan, h, w, 3, layout=layout)
        net.set_input_size(h, w)
        assert net.tensor_shapes == ref.tensor_shapes and net.flops_per_image == ref.flops_per_image
        assert [(hd['h'], hd['w']) for hd in net.heads] == [(hd['h'], hd['w']) for hd in ref.heads]
        b = 1 + i % 3
        assert_same(run(net, b, i), run(ref, b, i), f'{name} {h}x{w} batch {b}')
        if i % 4 == 1:
            assert_same(run(net, b, i, uint8=True), run(ref, b, i, uint8=True), f'{name} {h}x{w} uint8')
        ref.close()
    net.close()


# ---------------------------------------------------------------------------------------------------- host API
@pytest.mark.parametrize('name', tbm.NAMES)
def test_predictor_from_shell_equals_cifcaf_on_the_compiled_fields(name):
    shell = mm.calibrate_pose_heads(tbm.make_pose_shell(name, seed=5))
    pred = predictor.from_shell(shell, 161, 161, 4)
    assert pred.net.heads[0]['stride'] == 16 and (pred.net.heads[0]['h'], pred.net.heads[0]['w']) == (11, 11)
    images = torch.randn(4, 3, 161, 161, generator=torch.Generator().manual_seed(3)).pin_memory()
    sk = torch.tensor(shell.head_nets[1].meta.skeleton, dtype=torch.int64) - 1
    total = 0
    for b in (4, 3):
        res = pred.batch(images[:b])
        cif, caf = pred.fields_batch(images[:b].cuda())
        want = decoder.CifCaf(17, sk).decode_batch(cif, 16, caf, 16)
        assert len(res) == len(want) == b
        for (a, i), (wa, wi) in zip(res, want):
            assert torch.equal(a, wa) and torch.equal(i, wi)
            total += int(a.shape[0])
    print(name, 'annotations', total)
    pred.close()


@pytest.mark.parametrize('name', tbm.NAMES)
def test_det_predictor_from_shell_equals_cifdet_on_the_compiled_fields(name):
    shell = det_models.calibrate_det_head(det_models.make_det_shell(tbm.make_base(name), 91, 1, seed=2))
    pred = predictor.from_shell(shell, 161, 161, 3)
    assert isinstance(pred, predictor.DetPredictor)
    images = torch.randn(3, 3, 161, 161, generator=torch.Generator().manual_seed(4)).pin_memory()
    res = pred.batch(images)
    (field,) = pred.fields_batch(images.cuda())
    assert tuple(field.shape) == (3, 91, 6, 11, 11)
    want = decoder.CifDet(91).decode_batch(field, 16, nms=True)
    assert len(res) == len(want) == 3
    for (c, s, bx), (wc, ws, wb) in zip(res, want):
        assert torch.equal(c, wc) and torch.equal(s, ws) and torch.equal(bx, wb)
    pred.close()


# ---------------------------------------------------------------------------------------------------- plugin
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'oracle', '_ref_pkg')

SCRIPT = textwrap.dedent('''
    import json, os, sys, warnings
    warnings.filterwarnings('ignore')
    import numpy as np
    import torch
    import torchvision
    import openpifpaf
    from openpifpaf.network import basenetworks, factory
    torch.ops.openpifpaf.set_quiet(True)
    assert 'openpifpaf_b200' in openpifpaf.plugin.REGISTERED
    name = sys.argv[2]
    # from scratch: no checkpoint can be downloaded
    basenetworks.ShuffleNetV2.pretrained = False
    basenetworks.SqueezeNet.pretrained = False
    factory.BASE_FACTORIES['shufflenetv2x1'] = lambda: basenetworks.ShuffleNetV2(
        'shufflenetv2x1', lambda pretrained: torchvision.models.shufflenet_v2_x1_0(weights=None), 1024)
    factory.BASE_FACTORIES['squeezenet'] = lambda: basenetworks.SqueezeNet(
        'squeezenet', lambda pretrained: torchvision.models.squeezenet1_1(weights=None))
    sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
    import mobilenetv2_models

    torch.manual_seed(0)
    openpifpaf.network.Factory.base_name = name
    openpifpaf.network.Factory.checkpoint = None
    datamodule = openpifpaf.plugins.coco.CocoKp()
    predictor = openpifpaf.Predictor(head_metas=datamodule.head_metas)
    multi = predictor.processor
    (top,) = [d for d in multi.decoders if d is not None]
    assert type(top).__name__ == 'CifCafB200', type(top).__name__
    mobilenetv2_models.calibrate_pose_heads(predictor.model)
    ref = openpifpaf.decoder.CifCaf(predictor.model_cpu.head_metas[:1], predictor.model_cpu.head_metas[1:2])
    calls = []
    orig = type(top).batch
    def spy(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)
    type(top).batch = spy
    total = 0
    try:
        images = torch.randn(3, 3, 161, 161, generator=torch.Generator().manual_seed(3))
        got = multi.batch(predictor.model, images, device=predictor.device)
        (pred,) = [p for (_, _, p) in top._compiled.values()]
        cif, caf = [f.cpu() for f in pred.fields_batch(images.to(predictor.device))]
        for i in range(3):
            want = ref([cif[i], caf[i]])
            assert len(got[i]) == len(want), (i, len(got[i]), len(want))
            for a, b in zip(sorted(got[i], key=lambda a: -a.score), sorted(want, key=lambda a: -a.score)):
                assert abs(a.score - b.score) <= 1e-5
                assert np.abs(a.data[:, :2] - b.data[:, :2]).max() <= 1e-4
                assert np.abs(a.data[:, 2] - b.data[:, 2]).max() <= 1e-5
            total += len(want)
    finally:
        type(top).batch = orig
    assert calls and top._compiled
    print('PLUGIN_TORCHVISION_BACKBONE_OK', json.dumps({'base': name, 'annotations': total}))
''')


@pytest.mark.skipif(not os.path.exists(os.path.join(PKG, 'openpifpaf', '_cpp.so')),
                    reason='oracle/_ref_pkg not staged (python oracle/build_ref.py in the build container)')
@pytest.mark.parametrize('name', ['shufflenetv2x1', 'squeezenet'])
def test_reference_predictor_runs_through_the_plugin(name, tmp_path):
    env = dict(os.environ, PYTHONPATH=f'{PKG}:{ROOT}')
    r = subprocess.run([sys.executable, '-c', SCRIPT, ROOT, name], capture_output=True, text=True, env=env,
                       cwd=str(tmp_path), timeout=900)
    assert 'PLUGIN_TORCHVISION_BACKBONE_OK' in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout.strip().splitlines()[-1])
