"""Compile metagym_b200/csrc/*.cu into metagym_b200/libmgb200.so with nvcc for sm_90a (in-tree, no JIT cache)."""
import glob
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libmgb200.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]     # H100 (Hopper)

NVCC_FLAGS = GENCODE + [
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--use_fast_math=false",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libmgb200.so cannot be built (there is no CPU fallback)")


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(ROOT, "include", "mgb200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


# per-file extra flags: the maze renderer must reproduce float64 results of code that never fuses multiply-add
# quad.cu: every FMA is written out (fmaf / dot3 / det2) so that all kernel variants compute the same bits
# rnn_seq.cu: the forward runs the rollout's cell and must compile it exactly as maze.cu does
PER_FILE_FLAGS = {"maze.cu": ["-fmad=false"], "quad.cu": ["-fmad=false"], "rnn_seq.cu": ["-fmad=false"]}


def build(force=False, verbose=False):
    """Returns the path of the shared library, (re)building it when a source is newer."""
    if not force and not needs_build():
        return LIB
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
    objdir = os.path.join(PKG, "build")
    os.makedirs(objdir, exist_ok=True)
    log = ""
    objs = []
    inc = ["-I", os.path.join(ROOT, "include"), "-I", CSRC]
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [_nvcc()] + flags + PER_FILE_FLAGS.get(os.path.basename(src), []) + inc + ["-c", "-o", obj, src]
        res = subprocess.run(cmd, capture_output=True, text=True)
        log += " ".join(cmd) + "\n" + res.stdout + res.stderr
        if res.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + log)
        objs.append(obj)
    cmd = [_nvcc()] + GENCODE + ["-shared", "-o", LIB] + objs
    res = subprocess.run(cmd, capture_output=True, text=True)
    log += " ".join(cmd) + "\n" + res.stdout + res.stderr
    with open(os.path.join(PKG, "libmgb200.build.log"), "w") as f:
        f.write(log)
    if res.returncode != 0:
        raise RuntimeError("nvcc link failed:\n" + log)
    if verbose:
        print(log)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
