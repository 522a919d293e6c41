"""Build libstardist_b200.so (sm_90a) in-tree with nvcc.  Used by __graft_entry__.build()."""
import os, subprocess, sys, concurrent.futures as cf

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libstardist_b200.so")
OBJ = os.path.join(CSRC, "_obj")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default"]
# translation units; exact=True -> -fmad=false (bit-exact integer/float restatements of the reference)
UNITS = [
    ("runtime.cu", False), ("candidates.cu", True), ("nms2d.cu", True), ("nms2d_nv32.cu", True),
    ("nms2d_nv128.cu", True), ("label2d.cu", True), ("label3d.cu", True), ("blocks.cu", True), ("prep.cu", True), ("nms3d.cu", True), ("unet_simt.cu", False), ("unet_tc.cu", False), ("unet_exec.cu", False), ("overlap.cu", False),
    ("stardist.cu", True), ("labelprep.cu", True), ("traindata.cu", True),
    ("unet_train.cu", False), ("unet_train_tf32.cu", False), ("unet_train_bf16.cu", False), ("unet_any.cu", False), ("augment.cu", True), ("helpers.cu", True),
]

def _deps(src):
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(HERE, "..", "include", "stardist_b200.h"))
    return [src] + hs

def _stale(target, deps):
    if not os.path.exists(target): return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))

def _compile(unit):
    name, exact = unit
    src = os.path.join(CSRC, name); obj = os.path.join(OBJ, name.replace(".cu", ".o"))
    if not _stale(obj, _deps(src)): return obj, ""
    cmd = ["nvcc"] + ARCH + COMMON + (["-fmad=false"] if exact else []) + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (name, r.stdout, r.stderr))
    return obj, r.stderr

def build(verbose=False, extra_units=()):
    os.makedirs(OBJ, exist_ok=True)
    units = [u for u in UNITS if os.path.exists(os.path.join(CSRC, u[0]))] + list(extra_units)
    with cf.ThreadPoolExecutor(max_workers=8) as ex:
        objs = [o for o, _ in ex.map(_compile, units)]
    if _stale(OUT, objs):
        cmd = ["nvcc"] + ARCH + ["-shared", "-o", OUT] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    if verbose: print("built", OUT)
    return OUT

if __name__ == "__main__":
    build(verbose=True)
