"""Build libb200seg.so in-tree with nvcc for sm_90a (no torch dependency in the library)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200seg.so")
SOURCES = ["api.cu", "dice_ce.cu", "instnorm.cu", "pool_upsample.cu", "conv_direct.cu", "conv_tc.cu", "wgrad_tc.cu", "small_conv.cu", "biattn.cu", "dwconv.cu", "medformer_small.cu", "swin.cu", "swin_mma.cu", "optim.cu", "inference.cu", "surface.cu", "augment.cu", "attn_gate.cu", "attention.cu", "batchnorm.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC"]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "b200seg.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile every .cu into objects (parallel) and link the shared library."""
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, out.decode()))
        if verbose and out:
            print(out.decode())
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", LIB, *objs, *ARCH]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout.decode())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
