"""The fused MLP kernels keep their wgmma pipelined: ptxas must not serialise any wgmma of mlp_tc.cu for lack of
registers (warning C7512).  A serialised kernel waits for every MMA before issuing the next one, which leaves the tensor
cores idle between the MMAs of one weight item.  Cross-compiles mlp_tc.cu with the build's flags; needs nvcc, no GPU."""
import importlib.util
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "all-in-one-deflicker_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

pytestmark = pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")


def _build_flags():
    spec = importlib.util.spec_from_file_location("b200_build", os.path.join(CSRC, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.NVCC_FLAGS


def test_fused_kernels_wgmma_not_serialized(tmp_path):
    flags = _build_flags()
    assert "-v" in flags
    out = subprocess.run([NVCC] + flags + ["-c", os.path.join(CSRC, "mlp_tc.cu"), "-o", str(tmp_path / "mlp_tc.o")],
                         capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    kernels = set(re.findall(r"Compiling entry function '(_ZN4b200\d+tc_(?:fwd|bwd)_kernel\w+)'", log))
    assert len(kernels) == 12, sorted(kernels)           # six networks, forward and backward each
    serialized = [line for line in log.splitlines() if "C7512" in line]
    assert not serialized, "\n".join(serialized)
