"""CPU checks of the exact-data layer tests of the tensor-core convolutions (tests/convexact.py, tests/test_gpu_conv_exact.py):
the recipes keep every accumulator exact in fp32, the float64 references agree with float32 evaluations in other summation
orders on the very data the GPU tests use, a deliberately wrong reference differs from the right one on that data, and the
case tables reach every k_conv_wg instantiation under both accumulation schemes and every variant."""
import os
import numpy as np
import pytest

import convexact as CX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("case", CX.ALL_CASES, ids=CX.case_id)
def test_worst_case_bits_below_fp32(case):
    p = CX.PARAMS["fused" if case["family"] == "fused" else "conv"]
    bits = CX.worst_case_bits(p, CX.K_of(case))
    print(CX.case_id(case), {k: round(v, 2) for k, v in bits.items()})
    assert all(v < 22 for v in bits.values()), bits


@pytest.mark.parametrize("case", CX.STEM_CASES, ids=CX.case_id)
def test_stem_worst_case_bits_below_fp32(case):
    assert CX.stem_worst_case_bits(CX.PARAMS["stem"], case["cin"]) < 22


def _torch_conv_f32(D, nd, c0):
    """the same three products with torch's float32 convolution (its own summation order)"""
    import torch, torch.nn.functional as F
    conv = F.conv3d if nd == 3 else F.conv2d
    def t_x(a):
        x = torch.from_numpy(a.astype(np.float32))
        return x.permute(3, 0, 1, 2)[None] if nd == 3 else x.permute(0, 3, 1, 2)
    def t_w(a):
        cout, cin = a.shape[1], a.shape[2]
        return torch.from_numpy(a.astype(np.float32)).reshape(((3,) if nd == 3 else ()) + (3, 3, cout, cin)).permute(
            *((3, 4, 0, 1, 2) if nd == 3 else (2, 3, 0, 1)))
    xh, xl, wh, wl = t_x(D["x_hi"]), t_x(D["x_lo"]), t_w(D["w_hi"]), t_w(D["w_lo"])
    # one convolution over the three products stacked on the K axis
    y = conv(torch.cat([xh, xl, xh], 1), torch.cat([wh, wh, wl], 1), padding=1)
    y = y[0].permute(1, 2, 3, 0) if nd == 3 else y.permute(0, 2, 3, 1)
    return y.double().numpy()


@pytest.mark.parametrize("case", [c for c in CX.ALL_CASES if c["family"] != "heads"], ids=CX.case_id)
def test_conv_reference_is_order_independent(case):
    nd = 3 if case["family"] == "conv3d" else 2
    D = CX.gen_conv(case)
    ref = CX.conv_pre(D, nd, case["c0"])
    assert np.array_equal(_torch_conv_f32(D, nd, case["c0"]), ref)
    assert np.array_equal(CX.conv_pre(D, nd, case["c0"], order=-1, dtype=np.float32).astype(np.float64), ref)
    if case["family"] == "fused":
        logit, _, dist = CX.fused_ref(case, D)
        f32 = CX._bias_act(CX.conv_pre(D, 2, case["c0"], order=-1, dtype=np.float32), D, case["relu"], (), np.float32)
        o32 = f32 @ D["heads_w"]                                        # float32 matmul, then the float32 bias
        o32 = o32 + D["heads_b"]
        assert np.array_equal(o32[..., 32].astype(np.float64), logit)
        assert np.array_equal(o32[..., :case["R"]].astype(np.float64), dist)
    else:
        y = CX.conv_ref(case, D)
        hi, lo = CX.split16(y)
        assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), y), "hi + lo does not hold the output exactly"


@pytest.mark.parametrize("case", CX.HEADS_CASES, ids=CX.case_id)
def test_heads_reference_is_order_independent(case):
    import torch
    D = CX.gen_heads(case)
    _, dist = CX.heads_ref(D, case["R"])
    x = [torch.from_numpy(D[k].astype(np.float32)) for k in ("x_hi", "x_lo", "w_hi", "w_lo")]
    z = (torch.cat([x[0], x[1], x[0]], -1) @ torch.cat([x[2], x[2], x[3]], -1).t()) / D["w_scale"] + torch.from_numpy(D["bias"])
    assert np.array_equal(z[..., 1:case["R"] + 1].double().numpy(), dist)
    z2 = ((x[0] @ x[3].t() + x[1] @ x[2].t()) + x[0] @ x[2].t()) / D["w_scale"] + torch.from_numpy(D["bias"])
    assert np.array_equal(z2.double().numpy(), z.double().numpy())


@pytest.mark.parametrize("case", CX.STEM_CASES, ids=CX.case_id)
def test_stem_reference_is_order_independent(case):
    import torch, torch.nn.functional as F
    D = CX.gen_stem(case)
    y = CX.stem_ref(D, case["relu"])
    t = F.conv2d(torch.from_numpy(D["x"]).permute(0, 3, 1, 2), torch.from_numpy(D["w"]).permute(3, 2, 0, 1),
                 torch.from_numpy(D["bias"]), padding=1).permute(0, 2, 3, 1)
    if case["relu"]: t = torch.relu(t)
    assert np.array_equal(t.double().numpy(), y)
    hi, lo = CX.split16(y)
    assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), y)


def _mutant_rows():
    rows = []
    for fam, cases, muts in (("conv2d", CX.CONV2D_CASES, CX.CONV_MUTANTS), ("conv3d", CX.CONV3D_CASES, CX.CONV_MUTANTS),
                             ("heads", CX.HEADS_CASES, CX.HEADS_MUTANTS), ("fused", CX.FUSED_CASES, CX.FUSED_MUTANTS),
                             ("stem", CX.STEM_CASES, CX.STEM_MUTANTS)):
        for m in muts:
            if fam == "conv2d" and m == "dz_wrong":
                continue
            rows.append((fam, m))
    return rows


def _outputs(case, D, mutants=()):
    fam = case["family"]
    if fam in ("conv2d", "conv3d"):
        return [CX.conv_ref(case, D, mutants)]
    if fam == "heads":
        return list(CX.heads_ref(D, case["R"], mutants))
    if fam == "fused":
        return list(CX.fused_ref(case, D, mutants))
    return [CX.stem_ref(D, case["relu"], mutants)]


@pytest.mark.parametrize("family,mutant", _mutant_rows())
def test_mutants_are_detected(family, mutant):
    """every case of the family that can express the error catches it in at least one element: the data has teeth"""
    cases = {"conv2d": CX.CONV2D_CASES, "conv3d": CX.CONV3D_CASES, "heads": CX.HEADS_CASES, "fused": CX.FUSED_CASES,
             "stem": CX.STEM_CASES}[family]
    gen = {"heads": CX.gen_heads, "stem": CX.gen_stem}.get(family, CX.gen_conv)
    applicable = [c for c in cases if CX.mutant_applies(c, mutant)]
    assert applicable, "no %s case can express %s" % (family, mutant)
    for case in applicable:
        D = gen(case)
        good, bad = _outputs(case, D), _outputs(case, D, (mutant,))
        assert any(not np.array_equal(g, b) for g, b in zip(good, bad)), "%s not detected by %s" % (mutant, CX.case_id(case))
    print("%s / %s: detected in %d of %d cases" % (family, mutant, len(applicable), len(cases)))


def test_instance_coverage():
    """the case tables launch every k_conv_wg instantiation of unet_tc.cu, each under split_acc 0 and 1, and every family
    under variants 0, 1, 3 and 4"""
    src = CX.instances_in_source(os.path.join(ROOT, "stardist_b200", "csrc", "unet_tc.cu"))
    assert src == CX.ALL_INSTANCES, "unet_tc.cu instantiates %s; the tables model %s" % (sorted(src), sorted(CX.ALL_INSTANCES))
    reached = {}
    for c in CX.ALL_CASES:
        reached.setdefault(CX.instance(c), set()).add(c["split"])
    assert set(reached) == CX.ALL_INSTANCES, sorted(CX.ALL_INSTANCES - set(reached))
    for inst, splits in sorted(reached.items()):
        assert splits == {0, 1}, (inst, splits)
    for fam in ("conv2d", "conv3d", "heads", "fused"):
        assert {c["variant"] for c in CX.ALL_CASES if c["family"] == fam} == set(CX.VARIANTS), fam
    # the channel mixes, edges and switches each family is meant to exercise
    c2 = CX.CONV2D_CASES
    assert {(c["c0"], c["c1"]) for c in c2} == set(CX.MIXES_2D) and {c["cout"] for c in c2} == {32, 64, 128, 256}
    assert {(c["h"], c["w"]) for c in c2} >= set(CX.EDGES) and {c["n"] for c in c2} >= {1, 3}
    assert {c["relu"] for c in c2} == {0, 1} and {c["up"] for c in c2} == {0, 1}
    c3 = CX.CONV3D_CASES
    assert {c["d"] for c in c3} >= {1, 2, 3} and {c["cout"] for c in c3} == {32, 64, 128} and {c["up"] for c in c3} == {0, 2}
    hc = CX.HEADS_CASES
    assert {c["np"] for c in hc} == {48, 80, 112, 144} and {c["cfeat"] for c in hc} == {64, 128, 256} and {c["n"] for c in hc} == {1, 2}
    assert all(any(c["R"] == npd - 1 for c in hc if c["np"] == npd) and any(c["R"] < npd - 1 and c["R"] % 8 for c in hc if c["np"] == npd)
               for npd in (48, 80, 112, 144))
    fc = CX.FUSED_CASES
    assert {c["R"] for c in fc} == {1, 2, 7, 8, 9, 15, 16, 17, 31, 32} and {(c["c0"], c["c1"]) for c in fc} == {(0, 32), (0, 64), (32, 32)}
    assert {c["relu"] for c in fc} == {0, 1} and {c["n"] for c in fc} == {1, 2}
    # every family also has launches where each CTA of the persistent grid (132 on the H100) sweeps two or more tiles
    for fam in ("conv2d", "conv3d", "heads", "fused"):
        assert max(CX.n_tiles(c) for c in CX.ALL_CASES if c["family"] == fam and c["variant"] != 1) >= 2 * 132, fam
    print("k_conv_wg instances reached: %d/%d, each with split_acc 0 and 1" % (len(reached), len(CX.ALL_INSTANCES)))


def test_c_unet_create_refuses_configs_the_c_executor_cannot_run():
    """the C executor (csrc/unet_exec.cu) hard-codes ReLU, 3^d kernels, pool 2 and no batch norm; c_unet_create refuses any
    other config before it touches the device instead of running a different network"""
    import stardist_b200 as sd
    from stardist_b200 import _lib as L
    bad = [sd.Config2D(unet_activation='linear'), sd.Config2D(unet_last_activation='linear'), sd.Config2D(unet_batch_norm=True),
           sd.Config2D(unet_kernel_size=(5, 5)), sd.Config2D(unet_pool=(2, 1)),
           sd.Config3D(rays=sd.Rays_GoldenSpiral(16), unet_activation='elu'), sd.Config3D(rays=sd.Rays_GoldenSpiral(16), unet_pool=(1, 2, 2))]
    for cfg in bad:
        with pytest.raises(L.StarDistB200Error, match="C executor"):
            L.c_unet_create(cfg, {})
