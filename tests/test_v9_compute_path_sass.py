"""The compute warps of the LOAM-iVox batch kernel (p2plane_v9_kernel, fls_p2plane_v9.cu) keep their per-chunk path in
registers: between the ring pop and the `done` increment the common path — staged run, quantised top-6, LDL^T plane, DMMA —
touches no local memory.  The out-of-line rare paths (knn_scan_any, knn5_exact_any, plane_lstsq_qr) hand their results back
through the stack, so the only local loads allowed in that code are the ones right after such a call.

Two ways this has broken before, both invisible in the source: a result passed by reference to an out-of-line call kept
the hot path's copy on the stack, and the folder's inlined gn_step shared a stack slot with the compute warps' Jacobian,
which left every `J` store in local memory.  CPU only: compiles the kernel for sm_90a and reads the SASS."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "funny_lidar_slam_b200", "csrc")
SRC = os.path.join(CSRC, "fls_p2plane_v9.cu")


def _cuda_bin(tool):
    for d in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin"), "/usr/local/cuda/bin"):
        p = os.path.join(d, tool)
        if os.path.exists(p):
            return p
    return shutil.which(tool)


NVCC, NVDISASM = _cuda_bin("nvcc"), _cuda_bin("nvdisasm")


def _role_lines():
    """[first, last) source lines of the compute-warp branch of the kernel."""
    lines = open(SRC).read().splitlines()
    start = next(i for i, l in enumerate(lines, 1) if "=== compute warp" in l)
    end = next(i for i, l in enumerate(lines, 1) if "=== server warp" in l) - 1  # (the `else if` that opens the server)
    return start, end


@pytest.mark.skipif(NVCC is None or NVDISASM is None, reason="needs nvcc and nvdisasm")
def test_v9_compute_path_has_no_local_memory_traffic(tmp_path):
    cubin = tmp_path / "v9.cubin"
    subprocess.run([NVCC, "-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                    "-lineinfo", SRC, "-o", str(cubin)], check=True, cwd=CSRC, capture_output=True, text=True)
    sass = subprocess.run([NVDISASM, "-g", "-c", str(cubin)], check=True, capture_output=True, text=True).stdout
    start, end = _role_lines()

    in_kernel, where, since_call, seen, bad = False, None, 1 << 30, 0, []
    for line in sass.splitlines():
        m = re.match(r"^\$?([$\w]+):\s*$", line)
        if m and not m.group(1).startswith(".L"):
            # the kernel body is the label without a '$'-joined callee suffix
            in_kernel = "p2plane_v9_kernel" in m.group(1) and "$" not in m.group(1)
            continue
        m = re.match(r"\s*//## File \"([^\"]+)\", line (\d+)", line)
        if m:
            where = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        if not in_kernel or "*/" not in line or where is None:
            continue
        ins = line.split("*/", 1)[1].strip()
        if not ins or ins.startswith("/*"):
            continue
        since_call = 0 if re.search(r"\bCALL\b", ins) else since_call + 1
        f, ln = where
        compute = (f == "fls_p2plane_v9.cu" and start <= ln < end) or f in ("fls_plane.cuh", "fls_knn.cuh")
        if not compute:
            continue
        seen += 1
        if re.search(r"\bSTL\b", ins) or (re.search(r"\bLDL\b", ins) and since_call > 16):
            bad.append(f"{f}:{ln}: {ins}")
    assert seen > 500, "the compute-warp section was not found in the SASS"
    assert not bad, "local-memory traffic on the compute warps' path:\n" + "\n".join(bad[:40])
