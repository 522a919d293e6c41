"""CPU checks of the exact-data layer tests of the fp32 CUDA-core network kernels (tests/simtexact.py,
tests/test_gpu_simt_exact.py): the recipe keeps every accumulator exact in fp32, the float64 references agree with torch's
float32 evaluations on the very data the GPU tests use, a deliberately wrong reference differs from the right one on that
data, the case tables launch every kernel instance of unet_simt.cu, and they contain every launch class the CUDA-core
executors make for the shipped and the tensor-core-refused configurations."""
import os
import numpy as np
import pytest

import simtexact as SX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", [c for c in SX.ALL_CASES if SX.K_of(c)], ids=SX.case_id)
def test_worst_case_bits_below_fp32(case):
    bits = SX.worst_case_bits(SX.PARAMS, SX.K_of(case))
    assert bits < 24, bits
    if case["family"] == "class":                      # acc - max must be exact too
        assert SX.logit_bits(case) < 24


def test_largest_K_of_the_networks_is_in_the_tables():
    K = {f: max(SX.K_of(c) for c in SX.ALL_CASES if c["family"] == f) for f in ("conv", "stem", "generic")}
    print("largest K per family:", K, "bits:", {f: round(SX.worst_case_bits(SX.PARAMS, k), 2) for f, k in K.items()})
    assert K["conv"] >= 27 * 256 and K["generic"] >= 343 * 32


def _torch_conv_f32(case, D):
    """[upsample(lo), skip] through torch's float32 convolution: its own summation order"""
    import torch, torch.nn.functional as F
    x = D["skip"]
    if case["cin_lo"]:
        x = np.concatenate([SX.upsample_nd(D["lo"], case["up"]), x], -1)
    xt = torch.from_numpy(np.ascontiguousarray(x)).permute(0, 4, 1, 2, 3)
    wt = torch.from_numpy(D["w"]).permute(4, 3, 0, 1, 2)
    y = F.conv3d(xt, wt, torch.from_numpy(D["bias"]), padding=(case["kz"] // 2, 1, 1)).permute(0, 2, 3, 4, 1)
    return (torch.relu(y) if case["relu"] else y).double().numpy()


@pytest.mark.parametrize("case", SX.CONV_CASES + SX.STEM_CASES, ids=SX.case_id)
def test_conv3_reference_is_order_independent(case):
    D = SX.gen(case)
    assert np.array_equal(_torch_conv_f32(case, D), SX.conv3_ref(case, D))


@pytest.mark.parametrize("case", SX.GENERIC_CASES, ids=SX.case_id)
def test_generic_reference_is_torch_with_tf_padding(case):
    """torch's float32 conv3d on the input padded by (pad_total // 2, rest) with the kernel's stride"""
    import torch, torch.nn.functional as F
    D = SX.gen(case)
    pads = []
    for a, ax in enumerate("dhw"):
        _, total, before = SX.same_padding(case[ax], case["k"][a], case["s"][a])
        pads = [before, total - before] + pads                                  # F.pad lists the last axis first
    x = F.pad(torch.from_numpy(D["x"]).permute(0, 4, 1, 2, 3), pads)
    y = F.conv3d(x, torch.from_numpy(D["w"]).permute(4, 3, 0, 1, 2), torch.from_numpy(D["bias"]), stride=case["s"])
    y = y.permute(0, 2, 3, 4, 1)
    if case["relu"]: y = torch.relu(y)
    assert np.array_equal(y.double().numpy(), SX.generic_ref(case, D))


@pytest.mark.parametrize("case", SX.MAXPOOL_CASES[:3], ids=SX.case_id)
def test_maxpool_reference_is_a_window_max(case):
    D = SX.gen(case)
    n, d, h, w, c = D["x"].shape
    pz, py, px = case["pool"]
    want = D["x"].reshape(n, d // pz, pz, h // py, py, w // px, px, c).max(axis=(2, 4, 6))
    assert np.array_equal(SX.maxpool_ref(case, D), want)


@pytest.mark.parametrize("case", SX.HEADS_CASES[::5], ids=SX.case_id)
def test_heads_dist_is_exact_in_float32(case):
    D = SX.gen(case)
    _, dist = SX.heads_ref(case, D)
    assert np.array_equal((D["feat"] @ D["wd"] + D["bd"]).astype(np.float64), dist)


def test_class_head_bound():
    """the softmax bound grows by one ulp per output: C + 9 for every C the kernel takes"""
    for C in range(1, 33):
        assert SX.class_head_ulps(C) == C + 9, (C, SX.class_head_ulps(C))
    print("prob_class bound (float32 ulps of the float64 value):", {C: SX.class_head_ulps(C) for C in SX.CLASS_C})


# ------------------------------------------------------------------------------------------------ mutants
FAMILIES = {
    "conv": (SX.CONV_CASES, SX.CONV_MUTANTS), "stem": (SX.STEM_CASES, SX.STEM_MUTANTS),
    "generic": (SX.GENERIC_CASES, SX.GENERIC_MUTANTS), "maxpool": (SX.MAXPOOL_CASES, SX.MAXPOOL_MUTANTS),
    "heads": (SX.HEADS_CASES, SX.HEADS_MUTANTS), "class": (SX.CLASS_CASES, SX.CLASS_MUTANTS)}


def _caught(case, D, m):
    """the mutant's reference fails the comparison the GPU test makes against the right one"""
    fam = case["family"]
    if fam in ("conv", "stem"):
        return bool(SX.first_mismatch(SX.conv3_ref(case, D, (m,)), SX.conv3_ref(case, D), "out"))
    if fam == "generic":
        return bool(SX.first_mismatch(SX.generic_ref(case, D, (m,)), SX.generic_ref(case, D), "out"))
    if fam == "maxpool":
        return bool(SX.first_mismatch(SX.maxpool_ref(case, D, (m,)), SX.maxpool_ref(case, D), "out"))
    if fam == "heads":
        (pb, db), (pg, dg) = SX.heads_ref(case, D, (m,)), SX.heads_ref(case, D)
        return bool(SX.first_mismatch(db, dg, "dist") or SX.prob_mismatch(pb.astype(np.float32), pg))
    bad = SX.class_ref(case, D, (m,)).astype(np.float32)              # as a kernel with the error would store it
    return bool(SX.softmax_mismatch(bad, SX.class_ref(case, D), case["C"]))


@pytest.mark.parametrize("family,mutant", [(f, m) for f, (_, ms) in FAMILIES.items() for m in ms])
def test_mutants_are_detected(family, mutant):
    """a kernel with the error fails on at least one case of the family that can express it"""
    cases = FAMILIES[family][0]
    applicable = [c for c in cases if SX.mutant_applies(c, mutant)]
    assert applicable, "no %s case can express %s" % (family, mutant)
    caught = [c for c in applicable if _caught(c, SX.gen(c), mutant)]
    print("%s / %s: caught by %d of %d applicable cases" % (family, mutant, len(caught), len(applicable)))
    assert caught, "%s is not detected by any %s case" % (mutant, family)


# ------------------------------------------------------------------------------------------------ coverage
def test_instance_coverage():
    """a Python copy of sdb_conv3_nd's dispatch sends some case to every kernel instance unet_simt.cu launches"""
    src = SX.instances_in_source(os.path.join(ROOT, "stardist_b200", "csrc", "unet_simt.cu"))
    assert len(src) == 9, sorted(src)
    reached = {SX.instance(c) for c in SX.ALL_CASES} - {None}
    assert reached == src, "not reached: %s; not in the source: %s" % (sorted(src - reached), sorted(reached - src))
    print("unet_simt.cu instances reached: %d/%d: %s" % (len(reached & src), len(src), ", ".join(sorted(reached))))


def test_tables_contain_every_listed_value():
    conv = SX.CONV_CASES
    assert {c["cout"] for c in conv} >= set(SX.COUTS) and {(c["cin_skip"], c["cin_lo"]) for c in conv} >= set(SX.MIXES)
    assert {tuple(c["up"]) for c in conv if c["cin_lo"] and c["kz"] == 1} == set(SX.UPS[1])
    assert {tuple(c["up"]) for c in conv if c["cin_lo"] and c["kz"] == 3} == set(SX.UPS[3])
    assert {c["h"] for c in conv} >= {1, 15, 16, 17, 33, 130} and {c["w"] for c in conv} >= {1, 15, 16, 17, 33, 130}
    assert {c["d"] for c in conv if c["kz"] == 3} >= set(SX.DEPTHS) and {c["n"] for c in conv} == {1, 2, 3}
    assert {c["relu"] for c in conv} == {0, 1} and any(c["cin_skip"] + c["cin_lo"] > 16 and c["cin_lo"] for c in conv)
    stem = SX.STEM_CASES
    assert {(c["cin_skip"], c["cout"], c["kz"]) for c in stem} == {(a, b, k) for a in (1, 2, 3, 4) for b in (32, 64) for k in (1, 3)}
    npix = [c["n"] * c["d"] * c["h"] * c["w"] for c in stem]
    assert any(p > 128 and p % 128 for p in npix) and any(p == 16 * 64 * 64 for p in npix)
    gen = SX.GENERIC_CASES
    assert {(tuple(c["k"]), tuple(c["s"])) for c in gen} >= {(k, s) for k in SX.KERNELS for s in SX.STRIDES}
    assert {c["cin"] for c in gen} == {1, 8, 32} and {c["n"] for c in gen} == {1, 2} and {c["relu"] for c in gen} == {0, 1}
    pcs = {SX.pad_class(c[ax], c["k"][a], c["s"][a]) for c in gen for a, ax in enumerate("dhw")}
    assert pcs == {"0", "odd", "even"} and any(c[ax] == 1 for c in gen for ax in "dhw")
    assert any(c["d"] == 1 and c["k"][0] == 1 and c["s"][0] == 1 for c in gen)
    mp = SX.MAXPOOL_CASES
    assert {(tuple(c["pool"]), c["c"]) for c in mp} >= {(p, c) for p in SX.POOLS for c in (4, 32, 36)}
    assert max(c["n"] * c["d"] * c["h"] * c["w"] * c["c"] // (4 * int(np.prod(c["pool"]))) for c in mp) > SX.MAXPOOL_GRID
    assert max(c["size"] for c in SX.ADD_CASES) > SX.ADD_GRID
    assert {(c["R"], c["npix"]) for c in SX.HEADS_CASES} == {(r, p) for r in SX.HEADS_R for p in SX.HEADS_NPIX}
    cc = SX.CLASS_CASES
    assert {(c["C"], c["cf"]) for c in cc} == {(C, f) for C in SX.CLASS_C for f in (32, 128)} and all(c["npix"] % 128 for c in cc)


def _configs():
    import stardist_b200 as sd
    from stardist_b200.rays3d import rays_from_json
    from golden import demo3d
    rays_json, kwargs, _, _, _, _ = demo3d.load()
    return [
        ("Config2D()", sd.Config2D()),
        ("Config2D(grid=(2,1))", sd.Config2D(grid=(2, 1))),
        ("Config2D(grid=(1,2))", sd.Config2D(grid=(1, 2))),
        ("Config2D(grid=(4,2))", sd.Config2D(grid=(4, 2))),
        ("Config2D(n_channel_in=3)", sd.Config2D(n_channel_in=3)),
        ("Config2D(n_classes=3)", sd.Config2D(n_classes=3)),
        ("Config3D(unet_pool=(1,2,2))", sd.Config3D(unet_pool=(1, 2, 2))),
        ("Config3D(rays=Rays_GoldenSpiral(256))", sd.Config3D(rays=sd.Rays_GoldenSpiral(256))),
        ("3D_demo", sd.Config3D(rays=rays_from_json(rays_json), **kwargs)),
        ("Config3D(backbone='resnet', grid=(2,2,2), n_classes=2)", sd.Config3D(backbone='resnet', grid=(2, 2, 2), n_classes=2)),
    ]


def test_executor_coverage():
    """every (entry point, instance, up / pool / stride pattern, padding class) the CUDA-core executors launch for these
    configurations is a class of some case in the tables"""
    tables = {SX.case_class(c) for c in SX.ALL_CASES}
    missing = {}
    total = set()
    for name, cfg in _configs():
        launches = SX.executor_classes(cfg)
        total |= launches
        print("%s: %d launch classes" % (name, len(launches)))
        if launches - tables:
            missing[name] = sorted(launches - tables, key=str)
    assert not missing, "launch classes without a case: %s" % missing
    print("executor launch classes covered: %d/%d" % (len(total), len(total)))
