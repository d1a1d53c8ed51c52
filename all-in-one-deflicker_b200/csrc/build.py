"""Builds libb200deflicker.so (sm_90a) and libb200_hostcheck.so in-tree with nvcc / g++.

    python all-in-one-deflicker_b200/csrc/build.py [--force]

nvcc cross-compiles without a GPU.  The .so files are git-ignored but travel to the GPU box.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
LIB = os.path.join(PKG, "b200", "libb200deflicker.so")
HOSTLIB = os.path.join(PKG, "b200", "libb200_hostcheck.so")
CU = ["c_api.cu", "mlp_simt.cu", "atlas_kernels.cu", "mlp_tc.cu", "loss_heads.cu", "seg.cu", "eval_maps.cu", "eval_sse.cu", "producer.cu", "conv_simt.cu", "conv_tma.cu", "raft_kernels.cu", "corr_alt.cu", "stage2_io.cu", "png_encode.cu", "warp_error.cu", "blend.cu", "fidelity.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode()); h.update(f.read())
    return h.hexdigest()


def _sources():
    out = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cu", ".cuh", ".h", ".cpp", ".py"))]
    out.append(os.path.join(os.path.dirname(PKG), "include", "b200_deflicker.h"))
    return out


def build(force=False, verbose=False):
    stamp = os.path.join(HERE, ".build_stamp")
    dig = _digest(_sources())
    if (not force and os.path.exists(LIB) and os.path.exists(HOSTLIB) and os.path.exists(stamp)
            and open(stamp).read() == dig):
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    logs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for cu in CU:
        obj = os.path.join(HERE, "build", cu.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(HERE, cu), "-o", obj]
        procs.append((cu, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for cu, p in procs:
        out, _ = p.communicate()
        logs.append(f"==== {cu}\n{out}")
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {cu}")
    subprocess.check_call([nvcc, "-shared", NVCC_FLAGS[0], NVCC_FLAGS[1], "-o", LIB] + objs)
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", HOSTLIB,
                           os.path.join(HERE, "hostcheck.cpp")])
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(logs))
    if verbose:
        print("\n".join(logs))
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built", LIB)
