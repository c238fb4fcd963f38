"""Builds libmas_b200.so in-tree with nvcc for sm_90a (H100). No JIT cache: the library lives next to the package."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "build")
LIB = os.path.join(PKG, "lib", "libmas_b200.so")
SOURCES = ["norm.cu", "vq.cu", "vq_tc.cu", "contract_simt.cu", "conv4x4.cu", "lpips.cu", "contract_tc.cu", "conv_tma.cu", "gemm_tma.cu", "contract_tc3.cu", "edge.cu", "edge_quad.cu", "transformer.cu", "decode.cu", "attn.cu", "attn_fused.cu", "attn_causal.cu", "probe.cu", "capi.cu"]
NVCC_FLAGS = ["-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-Xcompiler", "-fPIC",
              "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [os.path.join(ROOT, "include", "mas_b200.h")]

    def one(src):
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + headers):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd), flush=True)
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        return o

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(one, SOURCES))
    if force or _stale(LIB, objs):
        r = subprocess.run([nvcc, "-shared", "-o", LIB] + objs + ["-lcudart"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
