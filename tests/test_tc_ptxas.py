"""The tensor-core convolution kernels compile without serialised wgmma groups and without new spills.

ptxas reports C7517 / C7519 / C7520 when it has to insert a warpgroup wait or arrive around a wgmma, because registers
the asynchronous MMA reads or writes are touched in between.  An injected wait retires the group in flight before the
next one can issue and an injected arrive splits a group, so the tensor cores idle; nothing but this report shows it.
Compiles conv_tc.cu and wgrad_tc.cu with the library's own flags (no GPU needed)."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "cbim-medical-image-segmentation_b200")

# spill bytes (stores, loads) per kernel of the shared-allocation kernels these replaced: conv_tc_kernel with every
# tile width inlined into one __global__, wgrad_tc_kernel without a register split.  No kernel may spill more.
SPILL_LIMIT = {"conv_tc_kernel": (948, 800), "wgrad_tc_kernel": (148, 272)}


def _build_module():
    spec = importlib.util.spec_from_file_location("_b200seg_build_ptxas", os.path.join(PKG, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _ptxas_report(src, tmp_path):
    nvcc = os.environ.get("NVCC", "nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("nvcc not found")
    b = _build_module()
    cmd = [nvcc, *b.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(b.CSRC, src), "-o", str(tmp_path / (src + ".o"))]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return r.stdout


def _kernels(report, kernel):
    """{mangled name: (spill stores, spill loads)} of every entry function whose name contains `kernel`"""
    out, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1) if kernel in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return out


@pytest.mark.parametrize("src,kernel", [("conv_tc.cu", "conv_tc_kernel"), ("wgrad_tc.cu", "wgrad_tc_kernel")])
def test_no_injected_warpgroup_sync_and_no_new_spills(src, kernel, tmp_path):
    report = _ptxas_report(src, tmp_path)
    injected = [l for l in report.splitlines() if re.search(r"\(C75(17|19|20)\)", l) and kernel in l]
    assert not injected, "ptxas serialises wgmma in %s:\n%s" % (kernel, "\n".join(injected[:10]))
    spills = _kernels(report, kernel)
    assert spills, "no %s in the ptxas report:\n%s" % (kernel, report[-2000:])
    st_max, ld_max = SPILL_LIMIT[kernel]
    over = {k: v for k, v in spills.items() if v[0] > st_max or v[1] > ld_max}
    assert not over, "%s spills more than %d / %d bytes (stores / loads): %s" % (kernel, st_max, ld_max, over)
