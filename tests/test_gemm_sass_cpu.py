"""Compiler-output checks of the wgmma kernel (sniper_b200/csrc/gemm_tc.cu), no GPU needed: every instantiation issues
its wgmma in groups of 4 of one shape behind a single warpgroup.arrive, so the tensor core's pipeline stays full within a
k-block.  A wgmma whose shape or accumulator registers are decided at run time makes ptxas serialise every instruction
(a C7519 note, one warpgroup.arrive and one gsb0 wait per HGMMA)."""
import os
import re
import shutil
import subprocess

import pytest

from sniper_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "sniper_b200", "csrc", "gemm_tc.cu")
pytestmark = pytest.mark.skipif(shutil.which("nvcc") is None or shutil.which("cuobjdump") is None,
                                reason="nvcc / cuobjdump not available")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("gemm_sass") / "gemm_tc.o")
    r = subprocess.run(["nvcc"] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-x", "cu", "-I", os.path.join(ROOT, "include"),
                                                     "-c", SRC, "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _kernels(sass):
    """{mangled name: [SASS instructions]} of every gemm_tc_kernel instantiation."""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "gemm_tc_kernel" in m.group(1) else None
            if cur:
                out[cur] = []
            continue
        ins = re.search(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", line)
        if cur and ins:
            out[cur].append(ins.group(1).strip())
    return out


def test_ptxas_reports_no_serialised_wgmma_and_no_spills(compiled):
    log, _ = compiled
    assert "C7519" not in log and "C7510" not in log, [l for l in log.splitlines() if "C75" in l][:4]
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(s == ("0", "0") for s in spills), spills


def test_mainloop_issues_wgmma_in_groups_of_four(compiled):
    _, sass = compiled
    kernels = _kernels(sass)
    # (tf32, bf16) x (K-major: 64, 128, 256, 256 + 64-column pieces, 256 + 128-column pieces; MN-major: 64, 128, 256)
    assert len(kernels) == 16, sorted(kernels)
    for name, code in kernels.items():
        seq = [i for i in code if i.startswith(("WARPGROUP.ARRIVE", "HGMMA"))]
        assert seq and seq[0].startswith("WARPGROUP.ARRIVE"), name
        groups = []
        for i in seq:
            if i.startswith("WARPGROUP.ARRIVE"):
                groups.append([])
            else:
                groups[-1].append(i)
        for grp in groups:
            # one warpgroup.arrive per 4 HGMMA of a single shape; only the last waits on the scoreboard (gsb0)
            assert len(grp) == 4, (name, grp)
            assert len({g.split()[0] for g in grp}) == 1, (name, grp)
            assert [("gsb0" in g) for g in grp] == [False, False, False, True], (name, grp)
        # one mainloop per width the kernel carries: the tile, and the tail pieces when it has them
        pieces = re.search(r"gemm_tc_kernelILi\dELi\dELi\d+ELi(\d+)E", name).group(1) != "0"
        assert len(groups) == (2 if pieces else 1), (name, len(groups))
