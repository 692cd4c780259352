"""conv_tc_kernel's wgmma schedule as ptxas compiles it (no GPU needed).

ptxas reports C7518 when it serialises wgmma.mma_async instructions (a wait after every MMA, because whether an
accumulator is still in flight depends on a divergent path) and C7517 when it injects a warpgroup.wait of its own
before registers written by an MMA are used.  Either one means the kernel does not run the asynchronous MMA chain its
consumer loop is written for, so the build of csrc/conv_tc.cu with the project's own flags must report neither."""
import os
import re
import shutil
import subprocess

import pytest

from object_detection_tracking_b200 import build


def _nvcc():
    cand = build._nvcc()
    return cand if os.path.exists(cand) or shutil.which(cand) else None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_conv_tc_wgmma_not_serialised(tmp_path):
    src = os.path.join(build.CSRC, "conv_tc.cu")
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "conv_tc.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    # every instantiation was compiled (fp16 / split / split + ACC, with and without swish, 64- and 128-column tiles)
    assert len(re.findall(r"Compiling entry function '\S*conv_tc_kernel", r.stdout)) == 12, r.stdout
    bad = [line for line in r.stdout.splitlines() if "C7517" in line or "C7518" in line]
    assert not bad, "\n".join(bad)
