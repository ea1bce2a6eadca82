"""The wgmma kernels keep their MMAs asynchronous.  When a wgmma sits on a path ptxas considers divergent, it inserts a
wait after every MMA (C7518: "wgmma.mma_async instructions are serialized") and warpgroup.arrive fences around the
accumulator registers (C7519): the kernel still computes the right result, only several times slower.  Compiled
with the library's own flags, for sm_90a; needs nvcc, not a GPU."""
import os
import subprocess

import pytest

from pillarnext_b200 import build

SOURCES = ["igemm.cu", "igemm_win.cu", "wgrad.cu"]


@pytest.mark.skipif(not os.path.exists(build.NVCC), reason="nvcc not found")
@pytest.mark.parametrize("src", SOURCES)
def test_wgmma_not_serialized(src, tmp_path):
    cmd = [build.NVCC] + build.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    log = r.stdout + r.stderr
    bad = [ln.strip() for ln in log.splitlines() if "C7518" in ln or "C7519" in ln]
    assert not bad, "%s: %d ptxas wgmma serialization diagnostics, first: %s" % (src, len(bad), bad[0][:300])
