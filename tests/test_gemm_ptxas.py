"""What ptxas makes of the wgmma GEMM kernels (no GPU needed): the MMAs of a K-block stay asynchronous and nothing spills.

ptxas serialises every wgmma of a kernel (a wait after each one, note C7518) when it cannot prove that the code around them is
uniform across the warpgroup.  Nothing fails then, and results stay the same; only the GEMMs get slower (DESIGN §3.3)."""
import os
import re
import shutil
import subprocess

import pytest

from vlfm_b200 import build


def test_gemm_wgmma_not_serialised_and_no_spills(tmp_path):
    if not shutil.which(build.NVCC) and not os.path.exists(build.NVCC):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "gemm_wgmma.cu")
    r = subprocess.run([build.NVCC, *build.FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "gemm_wgmma.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    serialised = [l for l in log.splitlines() if "C7518" in l]
    assert not serialised, "\n".join(serialised)
    # "Function properties for <kernel>" is followed by its stack / spill line
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    kernels = [p for p in props if "wgmma_kernel" in p[0]]
    assert len(kernels) >= 4
    for name, _, st, ld in kernels:
        assert st == "0" and ld == "0", f"{name} spills ({st} B stores, {ld} B loads)"
