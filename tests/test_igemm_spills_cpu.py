"""Every igemm_kernel instantiation fits its registers: the staged variants run 512 threads at 128 registers each (BN = 256
with setmaxnreg moving registers from the producer and store warpgroups to the consumers), so a spill there costs local-
memory traffic in the epilogue or the mainloop.  Compiled with the library's own flags, for sm_90a; needs nvcc, not a GPU."""
import os
import re
import subprocess

import pytest

from pillarnext_b200 import build


@pytest.mark.skipif(not os.path.exists(build.NVCC), reason="nvcc not found")
def test_igemm_kernels_do_not_spill(tmp_path):
    cmd = [build.NVCC] + build.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "igemm.cu"), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    spills, kernel, seen = [], None, 0
    for ln in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            kernel = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and kernel and "igemm_kernel" in kernel:
            seen += 1
            if int(m.group(1)) or int(m.group(2)):
                spills.append("%s: %s" % (kernel, ln.strip()))
            kernel = None
    assert seen >= 16, "expected the 16 igemm_kernel instantiations in the ptxas report, found %d" % seen
    assert not spills, "\n".join(spills)
