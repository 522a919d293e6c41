"""GPU parity tests of the 3D post-processing path (pytest -m gpu): NMS and label painting through
the reference-signature C ABI (_LIB_non_maximum_suppression_sparse / _LIB_polyhedron_to_label),
checked against the committed golden vectors (reference C++ run single-threaded) and, where
oracle/_ref is present, against the reference ext on fresh random inputs."""
import os, sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases
from oracle import ref_ext

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sd():
    import stardist_b200
    from stardist_b200 import _lib
    _lib.require_cuda()
    return stardist_b200


@pytest.fixture(scope="module")
def g3(golden_dir):
    return np.load(os.path.join(golden_dir, "nms3d.npz"))


@pytest.mark.parametrize("name", list(cases.NMS3D_CASES))
def test_nms3d_golden(sd, g3, name):
    from stardist_b200.lib.stardist3d import c_non_max_suppression_inds
    d, p, s, rays, thr, shape = cases.nms3d_inputs(name)
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    keep = c_non_max_suppression_inds(d, p, v, f, s, 1, 1, 0, thr)
    want = np.unpackbits(g3[name + "/keep"])[:len(d)].astype(bool)
    assert keep.dtype == np.bool_ and len(keep) == int(g3[name + "/n"])
    assert np.array_equal(keep, want), "%d decisions differ" % int((keep != want).sum())


@pytest.mark.parametrize("name", list(cases.NMS3D_CASES))
@pytest.mark.parametrize("mode", ["full", "kernel", "bbox", "full_overlap"])
def test_polyhedron_to_label_golden(sd, g3, name, mode):
    d, p, s, rays, thr, shape = cases.nms3d_inputs(name)
    keep = np.unpackbits(g3[name + "/keep"])[:len(d)].astype(bool)
    dk, pk, sk = d[keep], p[keep], s[keep]
    want = g3["%s/label_%s" % (name, mode)]
    kw = dict(mode="full", overlap_label=-1) if mode == "full_overlap" else dict(mode=mode)
    got = sd.polyhedron_to_label(dk, pk, rays, shape, prob=sk, verbose=False, **kw)
    assert got.dtype == np.int32 and got.shape == tuple(shape)
    ndiff = int((got != want).sum())
    lattice_aligned = cases.NMS3D_CASES[name][1] == 0.0      # noise 0: dist == 10 exactly, integer centres
    if lattice_aligned and mode in ("full", "full_overlap"):
        # Qhull's rounded facet planes decide voxels lying EXACTLY on a hull facet in the reference (hull conjunct of render
        # mode "full"); the product has no hull test.  No tolerance: every differing voxel must be such a voxel (rational
        # arithmetic, tests/hullcheck.py), labelled here and not by the reference.
        import hullcheck
        order = np.argsort(sk, kind='stable')[::-1]
        hullcheck.assert_only_exact_hull_boundary_voxels_differ(got, want, dk[order], pk[order], rays.vertices)
    else:
        assert ndiff == 0, "%d voxels differ" % ndiff


def test_nms3d_kdtree_and_bbox_flags_vs_reference(sd):
    if not ref_ext.available(): pytest.skip("oracle/_ref not present")
    os.environ["OMP_NUM_THREADS"] = "1"
    from stardist_b200.lib.stardist3d import c_non_max_suppression_inds
    rng = np.random.default_rng(5)
    rays = cases.rays_golden_spiral(32)
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    n = 1500
    p = rng.integers(0, 60, (n, 3)).astype(np.float32)
    d = (8 * (1 + .3 * rng.uniform(-1, 1, (n, 32)))).astype(np.float32)
    s = np.sort(rng.uniform(0, 1, n).astype(np.float32))[::-1].copy()
    for use_bbox, use_kd in ((1, 1), (1, 0), (0, 1)):
        want = ref_ext.stardist3d().c_non_max_suppression_inds(d, p, v, f, s, use_bbox, use_kd, 0, np.float32(.35))
        got = c_non_max_suppression_inds(d, p, v, f, s, use_bbox, use_kd, 0, np.float32(.35))
        assert np.array_equal(got, want), (use_bbox, use_kd, int((got != want).sum()))


def test_label3d_single_sphere_matches_reference_test_label(sd):
    """tests/test_nms3D.py:38-43 (test_label): one sphere of radius 20 with integer centre"""
    rays = cases.rays_golden_spiral(32)
    dist = 20 * np.ones((1, 32), np.float32)
    lbl = sd.polyhedron_to_label(dist, [[20, 20, 20]], rays, shape=(33, 44, 55), verbose=False)
    assert lbl.shape == (33, 44, 55) and lbl.max() == 1
    if ref_ext.available():
        v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
        want = ref_ext.stardist3d().c_polyhedron_to_label(dist, np.array([[20, 20, 20]], np.float32), v, f, np.array([1], np.int32),
                                                         np.int32(0), np.int32(0), np.int32(0), np.int32(0), (33, 44, 55))
        # lattice-aligned input: only voxels lying exactly on a hull facet may differ (tests/hullcheck.py, DESIGN.md)
        import hullcheck
        hullcheck.assert_only_exact_hull_boundary_voxels_differ(lbl, want, dist, np.array([[20, 20, 20]], np.float32), rays.vertices)


def test_empty_inputs_3d(sd):
    from stardist_b200.lib.stardist3d import c_non_max_suppression_inds
    rays = cases.rays_golden_spiral(16)
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    out = c_non_max_suppression_inds(np.zeros((0, 16), np.float32), np.zeros((0, 3), np.float32), v, f, np.zeros(0, np.float32), 1, 1, 0, np.float32(.4))
    assert out.shape == (0,)
    assert sd.polyhedron_to_label(np.zeros((0, 16)), np.zeros((0, 3)), rays, (5, 6, 7), verbose=False).shape == (5, 6, 7)


def test_unet3d_forward_vs_torch_fp32(sd, monkeypatch):
    import torch
    from oracle import unet_torch
    monkeypatch.setenv("STARDIST_B200_UNET", "simt")        # the exact-fp32 CUDA-core executor
    cfg = sd.Config3D(n_rays=16, rays=None) if False else sd.Config3D(rays=sd.Rays_GoldenSpiral(16))
    model = sd.StarDist3D(cfg, name=None, basedir=None)
    rng = np.random.default_rng(3)
    vol = rng.uniform(0, 1, (16, 32, 48)).astype(np.float32)
    x = torch.from_numpy(vol[None, ..., None]).cuda()
    prob, dist = model.net.forward(x)
    rp, rd = unet_torch.forward(cfg, model.weights, vol[None, ..., None])
    p, d = prob.cpu().numpy(), dist.cpu().numpy()
    assert p.shape == rp.shape and d.shape == rd.shape
    assert np.max(np.abs(p - rp)) <= 1e-5 * max(1.0, np.max(np.abs(rp)))
    assert np.max(np.abs(d - rd)) <= 1e-5 * max(1e-3, np.max(np.abs(rd))) + 1e-7


def test_predict_instances_3d_vs_oracle(sd):
    if not ref_ext.available(): pytest.skip("oracle/_ref not present")
    os.environ["OMP_NUM_THREADS"] = "1"
    from oracle import pipeline3d
    rays = sd.Rays_GoldenSpiral(24)
    cfg = sd.Config3D(rays=rays)
    model = sd.StarDist3D(cfg, name=None, basedir=None)
    # give the random-init net a usable dist head: bias 4.0 -> polyhedra of radius ~4 voxels
    k, b = model.weights['dist']; model.weights['dist'] = (k, b + np.float32(4.0)); model._net = None
    rng = np.random.default_rng(4)
    vol = rng.uniform(0, 1, (20, 40, 36)).astype(np.float32)
    prob, _ = model.predict(vol)
    pthr = float(np.quantile(prob, 0.97))
    labels, res = model.predict_instances(vol, prob_thresh=pthr, nms_thresh=0.3)
    ref_labels, ref = pipeline3d.predict_instances(cfg, rays, vol, pthr, 0.3, cand_from=model)
    assert labels.shape == vol.shape and len(res['prob']) > 2
    assert np.array_equal(res['points'], ref['points'])
    assert np.array_equal(res['prob'], ref['prob'])
    assert np.array_equal(res['dist'], ref['dist'])
    assert np.array_equal(labels, ref_labels)


def test_predict_3d_n_tiles_equals_untiled(sd):
    rng = np.random.default_rng(9)
    vol = rng.uniform(0, 1, (24, 72, 64)).astype(np.float32)
    model = sd.StarDist3D(sd.Config3D(rays=sd.Rays_GoldenSpiral(12)), name=None, basedir=None)
    p1, d1 = model.predict(vol)
    p2, d2 = model.predict(vol, n_tiles=(1, 3, 2))
    assert p1.shape == p2.shape
    assert np.max(np.abs(p1 - p2)) <= 1e-5 and np.max(np.abs(d1 - d2)) <= 1e-5 * max(1e-3, np.max(np.abs(d1))) + 1e-7


def test_resnet_forward_vs_torch_fp32(sd):
    """ResNet backbone (7^3 stem, strided block, 1^3 strided shortcut, residual adds) against the torch-CPU restatement,
    odd sizes (TensorFlow 'same' padding is asymmetric for even inputs with stride 2)"""
    import torch
    from oracle import unet_torch
    rays = sd.Rays_GoldenSpiral(8)
    for shape, grid in (((9, 20, 22), (1, 2, 2)), ((8, 17, 12), (2, 2, 2)), ((7, 9, 11), (1, 1, 1))):
        cfg = sd.Config3D(rays=rays, backbone='resnet', grid=grid, resnet_n_blocks=3)
        model = sd.StarDist3D(cfg, name=None, basedir=None)
        rng = np.random.default_rng(shape[1])
        vol = rng.uniform(0, 1, shape).astype(np.float32)
        x = torch.from_numpy(vol[None, ..., None]).cuda()
        prob, dist = model.net.forward(x)
        rp, rd = unet_torch.forward(cfg, model.weights, vol[None, ..., None])
        p, d = prob.cpu().numpy(), dist.cpu().numpy()
        assert p.shape == rp.shape and d.shape == rd.shape
        assert np.max(np.abs(p - rp)) <= 1e-5 * max(1.0, np.max(np.abs(rp)))
        assert np.max(np.abs(d - rd)) <= 1e-5 * max(1e-3, np.max(np.abs(rd))) + 1e-6


def test_reference_3d_demo_model_reproduces_reference_test(sd):
    """The reference's shipped 3D_demo checkpoint (tests/golden/demo3d.npz) on its test volume through the product path:
    (fp, tp, fn) == (0, 30, 21) as pinned by stardist tests/test_model3D.py:85-96, instances equal to the CPU oracle's."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import demo3d
    from oracle import pipeline3d
    from stardist_b200.utils import normalize
    from stardist_b200.matching import matching
    from stardist_b200.rays3d import rays_from_json
    rays_json, kwargs, weights, thr, img, mask = demo3d.load()
    rays = rays_from_json(rays_json)
    cfg = sd.Config3D(rays=rays, **kwargs)
    model = sd.StarDist3D(cfg, name=None, basedir=None, weights=weights)
    model.thresholds = dict(prob=thr['prob'], nms=thr['nms'])
    x = normalize(img, 1, 99.8)
    prob, dist = model.predict(x, n_tiles=(1, 2, 2))
    assert prob.shape == dist.shape[:3] and dist.shape[-1] == cfg.n_rays
    labels, res = model.predict_instances(x)
    assert labels.shape == img.shape[:3]
    st = matching(mask, labels, thresh=0.5)
    assert (st.fp, st.tp, st.fn) == demo3d.REFERENCE_TEST_STATS
    os.environ["OMP_NUM_THREADS"] = "1"
    ref_labels, ref = pipeline3d.predict_instances(cfg, rays, x, thr['prob'], thr['nms'], weights=weights)
    assert np.array_equal(res['points'], ref['points'])
    assert np.mean(labels != ref_labels) < 2e-3          # the oracle ran its own (torch-CPU) network: float-induced tolerance
    # the integer path on the trained model's real maps (cand_from=model): bit-equal
    labels2, res2 = model.predict_instances(x)
    ex_labels, ex = pipeline3d.predict_instances(cfg, rays, x, thr['prob'], thr['nms'], cand_from=model)
    assert np.array_equal(res2['points'], ex['points']) and np.array_equal(res2['prob'], ex['prob']) and np.array_equal(res2['dist'], ex['dist'])
    assert np.array_equal(labels2, ex_labels)



def test_multiclass_head_3d(sd):
    from oracle import unet_torch
    rng = np.random.default_rng(12)
    vol = rng.uniform(0, 1, (16, 40, 32)).astype(np.float32)
    for backbone in ('unet', 'resnet'):
        cfg = sd.Config3D(rays=sd.Rays_GoldenSpiral(12), n_classes=2, backbone=backbone)
        model = sd.StarDist3D(cfg, name=None, basedir=None)
        prob, dist, pc = model.predict(vol)
        rp, rd, rpc = unet_torch.forward(cfg, model.weights, vol[None, ..., None])
        assert pc.shape == prob.shape + (3,) and np.max(np.abs(pc - rpc[0])) <= 1e-5
        k, b = model.weights['dist']; model.weights['dist'] = (k, b + np.float32(3.0)); model._net = None
        prob, dist, pc = model.predict(vol)
        labels, res = model.predict_instances(vol, prob_thresh=float(np.quantile(prob, 0.97)), nms_thresh=0.3)
        assert res['class_prob'].shape == (len(res['prob']), 3)
        p = res['points']
        assert np.array_equal(res['class_prob'], pc[p[:, 0], p[:, 1], p[:, 2]])


@pytest.mark.parametrize("d,h,w,c0,c1,cout,relu,up2x", [(5, 12, 40, 0, 32, 32, 1, 0), (4, 9, 130, 0, 64, 64, 1, 0), (3, 6, 20, 32, 32, 32, 0, 0),
                                                        (4, 8, 16, 0, 64, 32, 1, 2), (6, 10, 24, 0, 32, 128, 1, 0), (2, 5, 200, 64, 64, 64, 1, 0)])
def test_conv3x3x3_tc_single_layer(d, h, w, c0, c1, cout, relu, up2x):
    """tensor-core 3x3x3 convolution (z planes as the tensor map's image axis, 27 taps) vs a float64 conv3d of the same split
    operands; two-source (concat) inputs and the 2x2x2 up-sampling epilogue"""
    import torch, torch.nn.functional as F
    from stardist_b200 import _lib as L
    from stardist_b200.models.unet_device import tc_weight_scale
    lib = L.require_cuda()
    g = torch.Generator(device='cpu').manual_seed(d * 131 + w + cout)
    cin = c0 + c1
    x = torch.randn((d, h, w, cin), generator=g).cuda()
    k = (torch.randn((3, 3, 3, cin, cout), generator=g) * (2.0 / (27 * cin)) ** 0.5).cuda()
    b = (torch.randn(cout, generator=g) * 0.1).cuda()
    hi = x.to(torch.float16); lo = (x - hi.float()).to(torch.float16)
    xs = torch.stack([hi, lo]).contiguous()
    x_eff = xs[0].double() + xs[1].double()
    ws = torch.empty((2, 27, cout, cin), dtype=torch.float16, device='cuda')
    wsc = tc_weight_scale(k.cpu().numpy())
    L.check(lib.sdb_split_weights_3d(L.ptr(k.contiguous()), cin, cout, wsc, L.ptr(ws[0]), L.ptr(ws[1]), L.stream_ptr()))
    k_eff = ((ws[0].double() + ws[1].double()) / wsc).reshape(3, 3, 3, cout, cin)          # [dz,dy,dx,cout,cin]
    src1 = xs[..., c0:].contiguous(); src0 = xs[..., :c0].contiguous() if c0 else None
    od, oh, ow = (2 * d, 2 * h, 2 * w) if up2x else (d, h, w)
    out = torch.zeros((2, od, oh, ow, cout), dtype=torch.float16, device='cuda')
    L.check(lib.sdb_conv3x3x3_tc(L.ptr(src0[0]) if c0 else L.ptr(None), L.ptr(src0[1]) if c0 else L.ptr(None), c0, L.ptr(src1[0]), L.ptr(src1[1]), c1,
                                 d, h, w, L.ptr(ws[0]), L.ptr(ws[1]), wsc, L.ptr(b), cout, relu, up2x, L.ptr(out[0]), L.ptr(out[1]), L.stream_ptr()))
    L.check(lib.sdb_tc_error_check(L.stream_ptr()))
    got = out[0].double() + out[1].double()
    y = F.conv3d(x_eff.permute(3, 0, 1, 2)[None], k_eff.permute(3, 4, 0, 1, 2), b.double(), padding=1)[0]
    if relu: y = F.relu(y)
    want = y.permute(1, 2, 3, 0)
    if up2x: want = want.repeat_interleave(2, 0).repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert (got - want).abs().max().item() <= 1e-5 * max(1.0, want.abs().max().item())


def test_unet3d_tc_vs_torch_fp32(sd):
    """3-D U-Net on the tensor cores against a float64 evaluation.  prob: 3e-7 of its scale.  dist of a RANDOM-INIT net is a
    near-cancelling sum (max ~0.07 from O(1) features): the split-fp16 / register-accumulated path leaves ~6e-7 absolute, i.e.
    7e-6 of that tiny scale with split_acc (1.2e-5 without; tests/tools/tc_split_error.py, DESIGN.md 5) -- the bound is
    1e-5 of max(map scale, feature scale 1) and 2e-5 of the map scale itself."""
    import torch
    from oracle import unet_torch
    from stardist_b200.models.unet_device import UNetDevice3DTC
    for shape, grid in (((16, 32, 48), (1, 1, 1)), ((8, 24, 136), (1, 2, 2))):
        cfg = sd.Config3D(rays=sd.Rays_GoldenSpiral(96), grid=grid)
        model = sd.StarDist3D(cfg, name=None, basedir=None)
        assert isinstance(model.net, UNetDevice3DTC)
        rng = np.random.default_rng(shape[2])
        vol = rng.uniform(0, 1, shape).astype(np.float32)
        prob, dist = model.net.forward(torch.from_numpy(vol[None, ..., None]).cuda())
        rp64, rd64 = unet_torch.forward(cfg, model.weights, vol[None, ..., None], dtype=torch.float64)
        p, dd = prob.cpu().numpy().astype(np.float64), dist.cpu().numpy().astype(np.float64)
        assert p.shape == rp64.shape and dd.shape == rd64.shape
        assert np.max(np.abs(p - rp64)) <= 1e-5 * max(1.0, np.max(np.abs(rp64)))
        err, scale = float(np.max(np.abs(dd - rd64))), float(np.max(np.abs(rd64)))
        assert err <= 1e-5 * max(1.0, scale) and err <= 2e-5 * scale, (err, scale)


@pytest.mark.parametrize("n,max_label,offset,density", [(0, 0, 1, 0.0), (1, 5, 1, 1.0), (1003, 17, 1, 0.5), (4096, 3000, 7, 0.2),
                                                         (100003, 5000, 1, 0.9), (65536, 40, 1, 1.0), (300001, 70000, 3, 0.3)])
def test_relabel_sequential_device_matches_host(sd, n, max_label, offset, density):
    """sdb_relabel_sequential == relabel_sequential (stardist/matching.py:319-406), bit-exact: relabelled map, forward map, count"""
    import torch
    from stardist_b200.matching import relabel_sequential, relabel_sequential_device
    rng = np.random.default_rng(n + max_label)
    present = np.flatnonzero(rng.uniform(size=max_label + 1) < density)
    present = present[present > 0]
    lab = (rng.choice(present, n) if len(present) else np.zeros(n, np.int64)).astype(np.int32)
    lab[rng.uniform(size=n) < 0.4] = 0
    t = torch.from_numpy(lab.copy()).cuda()
    out, fwd, cnt = relabel_sequential_device(t, offset=offset, max_label=max_label)
    if n == 0:
        assert cnt == 0; return
    want, wfwd, winv = relabel_sequential(lab, offset)
    assert np.array_equal(out.cpu().numpy(), want)
    assert cnt == len(winv) - offset
    assert np.array_equal(fwd.cpu().numpy()[:len(wfwd)], wfwd) and not fwd.cpu().numpy()[len(wfwd):].any()
    # already sequential input with offset 1: untouched
    t2 = torch.from_numpy(want.astype(np.int32)).cuda() if offset == 1 else None
    if t2 is not None:
        out2, _, cnt2 = relabel_sequential_device(t2)
        assert cnt2 == cnt and np.array_equal(out2.cpu().numpy(), want)


def test_relabel_sequential_device_rejects_negative(sd):
    import torch
    from stardist_b200.matching import relabel_sequential_device
    t = torch.tensor([0, 3, -1, 2], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        relabel_sequential_device(t, max_label=3)


def test_instances_from_prediction_sparse_points_3d(sd, g3):
    """StarDist3D._instances_from_prediction(points=...) (model3d.py:601-606, device-resident route) == golden NMS decisions
    + polyhedron_to_label + host relabel_sequential"""
    from stardist_b200.geometry.geom3d import polyhedron_to_label
    from stardist_b200.matching import relabel_sequential
    name = "r32_noise01_thr01"
    shape, noise, n_rays, pthr, nthr, seed, aniso = cases.NMS3D_CASES[name]
    prob, dist = cases.create_random_data_3d(shape, noise, n_rays, seed)
    mask = prob > pthr
    m2 = np.zeros_like(mask); m2[2:-2, 2:-2, 2:-2] = True
    mask &= m2
    points = np.stack(np.where(mask), axis=1)
    d = np.ascontiguousarray(dist[mask], np.float32); s = np.ascontiguousarray(prob[mask], np.float32)
    rays = cases.rays_golden_spiral(n_rays, aniso)
    model = sd.StarDist3D(sd.Config3D(rays=rays), name=None, basedir=None)
    labels, res = model._instances_from_prediction(shape, s, d, points=points, nms_thresh=float(nthr))
    ind = np.argsort(s, kind='stable')[::-1]
    keep = np.unpackbits(g3[name + "/keep"])[:len(d)].astype(bool)
    assert np.array_equal(res['points'], points[ind][keep])
    assert np.array_equal(res['prob'], s[ind][keep]) and np.array_equal(res['dist'], d[ind][keep])
    want = polyhedron_to_label(d[ind][keep], points[ind][keep], rays=rays, prob=s[ind][keep], shape=shape)
    want = relabel_sequential(want)[0]
    assert labels.dtype == np.int32 and np.array_equal(labels, want)


def test_relabel_sequential_device_reference_docstring_vectors(sd):
    """the known answers in the reference's docstring (stardist/matching.py:363-381) through sdb_relabel_sequential"""
    import torch
    from stardist_b200.matching import relabel_sequential_device
    lf = [1, 1, 5, 5, 8, 99, 42]
    out, fw, n = relabel_sequential_device(torch.tensor(lf, dtype=torch.int32, device="cuda"))
    assert out.cpu().tolist() == [1, 1, 2, 2, 3, 5, 4] and n == 5
    fw = fw.cpu().numpy()
    assert len(fw) == 100 and np.flatnonzero(fw).tolist() == [1, 5, 8, 42, 99] and fw[[1, 5, 8, 42, 99]].tolist() == [1, 2, 3, 4, 5]
    out5, _, _ = relabel_sequential_device(torch.tensor(lf, dtype=torch.int32, device="cuda"), offset=5)
    assert out5.cpu().tolist() == [5, 5, 6, 6, 7, 9, 8]
    with pytest.raises(ValueError):
        relabel_sequential_device(torch.tensor(lf, dtype=torch.int32, device="cuda"), offset=0)


@pytest.mark.parametrize("noise,n_rays", cases.NMS3D_ACCURACY_CASES)
def test_reference_nms_accuracy_property(sd, noise, n_rays):
    """the reference's own test_nms_accuracy (tests/test_nms3D.py:60-83) through the product path (list / float64 inputs
    as there): rendered IoU of two polyhedra, NMS at 0.95*iou keeps one, at 1.05*iou keeps both.  With oracle/_ref the rendered
    masks are compared with the reference's: the polar rays of the golden spiral get dist == 10.0 exactly here (sin(2 pi * +-1),
    sin(0)), so each polyhedron has vertices ON the voxel lattice -- the documented hull-facet caveat (DESIGN.md 5, 3D labels:
    the reference ANDs a Qhull hull test whose last-bit plane rounding decides such a voxel).  The bound asserted here is 0.1 % (these polyhedra have radius ~10)."""
    from stardist_b200.geometry.geom3d import polyhedron_to_label
    from stardist_b200.nms import non_maximum_suppression_3d_sparse
    dist, points, prob, rays, shape = cases.nms3d_accuracy_inputs(noise, n_rays)
    pts = [tuple(int(v) for v in p) for p in points]
    mask1 = polyhedron_to_label([dist[0]], [pts[0]], rays, shape=shape, verbose=False)
    mask2 = polyhedron_to_label([dist[1]], [pts[1]], rays, shape=shape, verbose=False)
    iou = np.count_nonzero(mask1 * mask2) / min(np.count_nonzero(mask1), np.count_nonzero(mask2) + 1e-10)
    sup1 = non_maximum_suppression_3d_sparse(dist, [1, .5], pts, rays=rays, nms_thresh=0.95 * iou, verbose=False)[0]
    sup2 = non_maximum_suppression_3d_sparse(dist, [1, .5], pts, rays=rays, nms_thresh=1.05 * iou, verbose=False)[0]
    assert len(sup1) == 1 and len(sup2) == 2
    if ref_ext.available():
        from oracle import pipeline3d
        for m, k in ((mask1, 0), (mask2, 1)):
            ref = pipeline3d.polyhedron_to_label(dist[k:k + 1], points[k:k + 1], rays, shape, prob[k:k + 1])
            import hullcheck
            nd = hullcheck.assert_only_exact_hull_boundary_voxels_differ((m > 0).astype(np.int32), (ref > 0).astype(np.int32), dist[k:k + 1], points[k:k + 1],
                                                                         rays.vertices, max_voxels=4)
            assert nd <= 2


@pytest.mark.parametrize("name", list(cases.NMS3D_CASES))
def test_nms3d_golden_other_kernel_paths(sd, g3, name):
    """the goldens through the non-default code paths: volumes on un-normalised planes (variant 0, the round-1 formulation),
    all heavy stages in one launch (split 0: reference stage order S3 -> S4 -> S5, hulls inside the CTA)"""
    from stardist_b200 import _lib
    from stardist_b200.lib.stardist3d import c_non_max_suppression_inds
    d, p, s, rays, thr, shape = cases.nms3d_inputs(name)
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    lib = _lib.load()
    want = np.unpackbits(g3[name + "/keep"])[:len(d)].astype(bool)
    try:
        for variant, split, bound in ((0, 1, 1), (1, 0, 1), (0, 0, 0), (1, 3, 1), (1, 1, 2)):      # split 3: CTA-per-pair S3 bound; bound 2: coarse fan
            lib.sdb_nms3d_set_variant(variant); lib.sdb_nms3d_set_split(split); lib.sdb_nms3d_set_s3_bound(bound)
            keep = c_non_max_suppression_inds(d, p, v, f, s, 1, 1, 0, thr)
            assert np.array_equal(keep, want), "(variant %d, split %d, bound %d): %d decisions differ" % (variant, split, bound, int((keep != want).sum()))
    finally:
        lib.sdb_nms3d_set_variant(1); lib.sdb_nms3d_set_split(1); lib.sdb_nms3d_set_s3_bound(1)


def _random_polyhedra(rng, n, n_rays, shape, aniso=None):
    rays = cases.rays_golden_spiral(n_rays, aniso)
    p = np.stack([rng.integers(4, s - 4, n) for s in shape], 1).astype(np.float32)
    d = (6 * (1 + .3 * rng.uniform(-1, 1, (n, n_rays)))).astype(np.float32)
    return rays, d, p


@pytest.mark.parametrize("n_rays,aniso", [(32, None), (96, (2, 1, 1))])
def test_polyhedron_to_label_mode_hull_vs_reference(sd, n_rays, aniso):
    """render mode "hull" (stardist3d_impl.cpp:1483-1486: Qhull facet planes) on generic float input, where no voxel lies
    within rounding distance of a facet: gift-wrapped facets give the same voxels"""
    if not ref_ext.available(): pytest.skip("oracle/_ref not present")
    from stardist_b200.lib.stardist3d import c_polyhedron_to_label
    rng = np.random.default_rng(11)
    shape = (40, 48, 56)
    rays, d, p = _random_polyhedra(rng, 40, n_rays, shape, aniso)
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    lab = np.arange(1, len(d) + 1, dtype=np.int32)
    for mode in (2, 0, 1):
        want = ref_ext.stardist3d().c_polyhedron_to_label(d, p, v, f, lab, np.int32(mode), np.int32(0), np.int32(0), np.int32(0), shape)
        got = c_polyhedron_to_label(d, p, v, f, lab, mode, 0, 0, 0, shape)
        assert np.array_equal(got, want), (mode, int((got != want).sum()))


@pytest.mark.parametrize("use_overlap,overlap_label,zero_labels", [(0, 0, True), (1, -1, True), (1, 0, False), (1, 0, True), (1, 7, True)])
def test_polyhedron_to_label_zero_labels_and_zero_overlap_label(sd, use_overlap, overlap_label, zero_labels):
    """labels == 0 (paints nothing and is painted over) and overlap_label == 0 make the reference's in-place rule
    (stardist3d_impl.cpp:1508-1517) depend on the whole cover sequence; the sequential variant reproduces it exactly"""
    if not ref_ext.available(): pytest.skip("oracle/_ref not present")
    from stardist_b200.lib.stardist3d import c_polyhedron_to_label
    rng = np.random.default_rng(12)
    shape = (28, 36, 40)
    rays, d, p = _random_polyhedra(rng, 60, 32, shape)          # dense enough for triple overlaps
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    lab = np.arange(1, len(d) + 1, dtype=np.int32)
    if zero_labels:
        lab[rng.random(len(lab)) < 0.3] = 0
    want = ref_ext.stardist3d().c_polyhedron_to_label(d, p, v, f, lab, np.int32(0), np.int32(0), np.int32(use_overlap), np.int32(overlap_label), shape)
    got = c_polyhedron_to_label(d, p, v, f, lab, 0, 0, use_overlap, overlap_label, shape)
    assert (want != 0).sum() > 1000
    assert np.array_equal(got, want), int((got != want).sum())


def test_c_entry_points_raise_instead_of_aborting(sd):
    """limits the reference does not have (256 rays / 512 faces) surface as exceptions, and a failing call through the
    void reference-signature ABI leaves the process alive with the message in sdb_last_error()"""
    import ctypes
    from stardist_b200 import _lib as L
    from stardist_b200.lib.stardist3d import c_non_max_suppression_inds, c_polyhedron_to_label
    rays = cases.rays_golden_spiral(300)
    v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
    d = np.ones((2, 300), np.float32); p = np.zeros((2, 3), np.float32)
    with pytest.raises(ValueError):
        c_non_max_suppression_inds(d, p, v, f, np.ones(2, np.float32), 1, 1, 0, np.float32(.4))
    with pytest.raises(ValueError):
        c_polyhedron_to_label(d, p, v, f, np.array([1, 2], np.int32), 0, 0, 0, 0, (8, 8, 8))
    # straight through the C ABI: result zeroed, error string set, no abort
    lib = L.load()
    res = np.ones(2, np.bool_)
    fn = lib._LIB_non_maximum_suppression_sparse
    fn.restype = None
    fn.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + [ctypes.c_float] + [ctypes.c_int] * 3 + [ctypes.c_void_p]
    fn(L.ptr(np.ones(2, np.float32)), L.ptr(d), L.ptr(p), 2, 300, len(f), L.ptr(v), L.ptr(f), 0.4, 1, 1, 0, L.ptr(res))
    assert not res.any() and b"unsupported" in lib.sdb_last_error()


def test_tied_scores_sparse_equals_dense_3d(sd):
    """overlapping survivors with EQUAL scores: the device (sparse) path paints in the order geom3d.polyhedron_to_label
    defines (argsort(prob, stable)[::-1]), so sparse == dense also on ties"""
    rays = sd.Rays_GoldenSpiral(32)
    cfg = sd.Config3D(rays=rays)
    model = sd.StarDist3D(cfg, name=None, basedir=None)
    shape = (24, 40, 40)
    rng = np.random.default_rng(3)
    pts = np.array([[12, 12, 12], [12, 15, 14], [12, 26, 26], [12, 24, 29], [10, 20, 20]])
    prob = np.array([.9, .9, .9, .9, .5], np.float32)            # two tied, overlapping pairs
    dist = (7 * (1 + .1 * rng.uniform(-1, 1, (5, 32)))).astype(np.float32)
    l_sparse, r_sparse = model._instances_from_prediction(shape, prob, dist, points=pts, nms_thresh=0.9)
    from stardist_b200.geometry.geom3d import polyhedron_to_label
    from stardist_b200.matching import relabel_sequential
    want = relabel_sequential(polyhedron_to_label(r_sparse['dist'], r_sparse['points'], rays, shape, prob=r_sparse['prob'], verbose=False))[0]
    assert len(r_sparse['prob']) == 5 and np.array_equal(l_sparse, want)


def test_paint3d_sphere_culling_is_result_neutral(sd):
    """k_paint3d skips bounding-box voxels outside the vertex ball / inside the kernel's inscribed ball (margins far above
    the rounding of the tests they short-cut): label maps with and without the culling are identical, incl. degenerate
    polyhedra (rays clamped to 1e-3), strong anisotropy and the reference's lattice-aligned test shapes"""
    from stardist_b200 import _lib
    from stardist_b200.lib.stardist3d import c_polyhedron_to_label
    lib = _lib.load()
    rng = np.random.default_rng(21)
    shape = (36, 48, 52)
    sets = []
    for n_rays, aniso in ((32, None), (96, (2, 1, 1)), (64, (1, 1.5, 4))):
        rays, d, p = _random_polyhedra(rng, 50, n_rays, shape, aniso)
        d2 = d.copy(); d2[rng.random(d2.shape) < 0.3] = 1e-3          # spikes / collapsed rays
        d3 = np.full_like(d, 5.0)                                       # lattice aligned
        sets += [(rays, d, p), (rays, d2, p), (rays, d3, p), (rays, (d * 0.05).astype(np.float32), p)]
    for rays, d, p in sets:
        v = np.ascontiguousarray(rays.vertices, np.float32); f = np.ascontiguousarray(rays.faces, np.int32)
        lab = np.arange(1, len(d) + 1, dtype=np.int32)
        for mode, ov in ((0, 0), (1, 0), (0, 1)):
            try:
                lib.sdb_label3d_set_cull(0)
                a = c_polyhedron_to_label(d, p, v, f, lab, mode, 0, ov, -1, shape)
                for cull in (1, 2, 3):          # sphere culling, direction bins, both (default)
                    lib.sdb_label3d_set_cull(cull)
                    b = c_polyhedron_to_label(d, p, v, f, lab, mode, 0, ov, -1, shape)
                    assert np.array_equal(a, b), (mode, ov, cull, int((a != b).sum()))
            finally:
                lib.sdb_label3d_set_cull(3)


def test_sparse_slab_forward_equals_dense_forward(sd, monkeypatch):
    """large-volume path (features + heads slab by slab, compact dist store; no dense dist map): same candidates, same
    instances and labels as the dense path, bit for bit, incl. a depth that is not a multiple of the slab"""
    import bench_data
    cfg = bench_data.bench_config_3d(96)
    model = sd.StarDist3D(cfg, name=None, basedir=None, weights=bench_data.bench_weights_3d(cfg))
    vol, _ = bench_data.synthetic_volume((40, 96, 128), seed=5, cell=(40, 96, 128))
    monkeypatch.setenv("STARDIST_B200_SPARSE_FORWARD", "0")
    l0, r0 = model.predict_instances(vol, prob_thresh=0.7, nms_thresh=0.3)
    p0 = model._last_maps()[0]
    monkeypatch.setenv("STARDIST_B200_SPARSE_FORWARD", "1")
    l1, r1 = model.predict_instances(vol, prob_thresh=0.7, nms_thresh=0.3)
    p1 = model._last[0].cpu().numpy()
    assert len(r0['prob']) > 20
    assert np.array_equal(p0, p1)
    for k in ('prob', 'points', 'dist'):
        assert np.array_equal(r0[k], r1[k]), k
    assert np.array_equal(l0, l1)
