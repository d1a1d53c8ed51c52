"""The fused backward kernels form their bias gradients (and the mapping's dW0) as row sums on the tensor cores, with
no shared-memory atomics and no per-value shuffle reductions.  A float atomicAdd to shared memory compiles to a
compare-and-swap spin loop (ATOMS.CAST.SPIN) on sm_90, and the shuffle trees it replaced ran in the epilogue, where a
warpgroup issues no MMA.  Cross-compiles mlp_tc.cu with the build's flags and reads the SASS; needs nvcc, no GPU."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "all-in-one-deflicker_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)),
                                reason="nvcc / cuobjdump not available")

# What stays per instance: the output layer's bias (one warp sum per output column and tile), and in the atlas the
# input gradient's quad sums and its max reduction.  The shuffle column sums needed 394 to 970.
MAX_SHFL_BFLY = 64


def _build_flags():
    spec = importlib.util.spec_from_file_location("b200_build", os.path.join(CSRC, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.NVCC_FLAGS


def test_backward_reductions_have_no_shared_atomics(tmp_path):
    obj = tmp_path / "mlp_tc.o"
    out = subprocess.run([NVCC] + _build_flags() + ["-c", os.path.join(CSRC, "mlp_tc.cu"), "-o", str(obj)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    sass = subprocess.run([CUOBJDUMP, "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    counts = {}
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        name = block.split("\n", 1)[0].strip()
        if "tc_bwd_kernel" in name:
            counts[name] = (block.count("ATOMS.CAST.SPIN"), block.count("SHFL.BFLY"))
    assert len(counts) == 6, sorted(counts)              # six networks
    bad = {n: c for n, c in counts.items() if c[0] != 0 or c[1] > MAX_SHFL_BFLY}
    assert not bad, bad
