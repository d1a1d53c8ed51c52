"""The fused forward kernels take their bias, first-layer and output-layer constants from shared memory: between a tile's
first HGMMA and the global store of its output rows y no instance issues a global load (LDG), and the plain mappings
(the flagship step's largest kernel) touch no local memory there either.  While a warpgroup runs its epilogue it issues
no MMA, so every such instruction is tensor-core idle time.  Total spill bytes stay at or below what each instance
spilled when the epilogues read the parameters from global memory.  Cross-compiles mlp_tc.cu with the build's flags and
reads the SASS; needs nvcc, no GPU."""
import importlib.util
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "all-in-one-deflicker_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)),
                                reason="nvcc / cuobjdump not available")

# (spill store bytes, spill load bytes) per instance when the epilogues read their constants with __ldg
SPILL_LIMITS = {
    "tc_fwd_kernelILb0ELi6ELi0E": (252, 268),     # plain mapping, 6 layers
    "tc_fwd_kernelILb0ELi4ELi0E": (252, 268),     # plain mapping, 4 layers
    "tc_fwd_kernelILb1ELi8ELi0E": (252, 332),     # atlas
    "tc_fwd_kernelILb1ELi8ELi1E": (204, 224),     # alpha
    "tc_fwd_kernelILb1ELi6ELi2E": (80, 136),      # position-encoded mapping, 6 layers
    "tc_fwd_kernelILb1ELi4ELi2E": (80, 136),      # position-encoded mapping, 4 layers
}
NO_LOCAL_IN_LOOP = ("tc_fwd_kernelILb0ELi6ELi0E", "tc_fwd_kernelILb0ELi4ELi0E")


def _build_flags():
    spec = importlib.util.spec_from_file_location("b200_build", os.path.join(CSRC, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.NVCC_FLAGS


def _key(name):
    for k in SPILL_LIMITS:
        if k in name:
            return k
    return None


def _tile_loop_loads(block):
    """LDG / LDL / STL from a tile's first HGMMA to the store of its output rows (a 32-bit STG: the flag words are
    16-bit stores, the positional-encoding image rows 128-bit ones)."""
    found, inside = [], False
    for addr, text in re.findall(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", block):
        op = text.split()[1] if text.startswith("@") else text.split()[0]
        if op.startswith("HGMMA"):
            inside = True
        elif inside and op.startswith(("LDG", "LDL", "STL")):
            found.append((addr, text.strip()))
        elif op.startswith("STG") and ".U16" not in op and ".128" not in op:
            inside = False
    return found


def test_forward_epilogues_read_no_global_memory(tmp_path):
    obj = tmp_path / "mlp_tc.o"
    out = subprocess.run([NVCC] + _build_flags() + ["-c", os.path.join(CSRC, "mlp_tc.cu"), "-o", str(obj)],
                         capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    spills = {}
    for name, st, ld in re.findall(r"Compiling entry function '(\w+)'.*?\n.*?\n\s*\d+ bytes stack frame, (\d+) bytes "
                                   r"spill stores, (\d+) bytes spill loads", log):
        if _key(name) and "tc_fwd_kernel" in name:
            spills[_key(name)] = (int(st), int(ld))
    assert sorted(spills) == sorted(SPILL_LIMITS), spills
    over = {k: v for k, v in spills.items() if v[0] > SPILL_LIMITS[k][0] or v[1] > SPILL_LIMITS[k][1]}
    assert not over, over

    sass = subprocess.run([CUOBJDUMP, "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    seen = set()
    for block in re.split(r"\n\s*Function : ", sass)[1:]:
        name = block.split("\n", 1)[0].strip()
        k = _key(name)
        if not k or "tc_fwd_kernel" not in name:
            continue
        seen.add(k)
        assert "HGMMA" in block, name
        loads = _tile_loop_loads(block)
        glob = [x for x in loads if x[1].split()[0].startswith("LDG") or " LDG" in x[1]]
        assert not glob, (name, glob[:8])
        if k in NO_LOCAL_IN_LOOP:
            assert not loads, (name, loads[:8])
    assert seen == set(SPILL_LIMITS), seen
