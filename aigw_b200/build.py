"""Build libaigw_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libaigw_b200.so")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
SOURCES = ["lib.cu", "chat_kernel.cu", "chat_walk.cu", "chat_walk_g0.cu", "chat_walk_g1.cu", "chat_walk_g2.cu", "chat_walk_g3.cu", "chat_walk_g4.cu", "chat_walk_g5.cu", "chat_walk_g6.cu", "chat_walk_g7.cu", "chat_walk_g8.cu", "chat_walk_g9.cu", "chat_small_g0.cu", "chat_small_g1.cu", "chat_small_g2.cu", "chat_small_g3.cu", "chat_small_g4.cu", "chat_small_g5.cu", "chat_small_g6.cu", "chat_small_g7.cu", "chat_small_g8.cu", "chat_small_g9.cu", "sse_kernel.cu", "bedrock_stream_kernel.cu", "stream_kernel.cu", "bpe_kernel.cu", "emb_kernel.cu", "mutate_kernel.cu", "batcher.cu", "sha256_kernel.cu", "cel_kernel.cu"]


def nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))] + [os.path.join(HERE, "..", "include", "aigw_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """One nvcc -c per source, in parallel (chat_kernel.cu alone takes minutes: six size classes of three kernels), then one link."""
    if not force and not needs_build():
        return SO
    from concurrent.futures import ThreadPoolExecutor
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    base = [nvcc()] + GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]
    if verbose:
        base.insert(1, "-Xptxas=-v")
    hdr_t = max(os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) if os.listdir(CSRC) else 0
    hdr_t = max(hdr_t, os.path.getmtime(os.path.join(HERE, "..", "include", "aigw_b200.h")))

    def one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        path = os.path.join(CSRC, src)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(path), hdr_t):
            cmd = base + ["-c", path, "-o", obj]
            if verbose:
                print(" ".join(cmd), file=sys.stderr)
            subprocess.check_call(cmd)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 2)) as ex:
        objs = list(ex.map(one, SOURCES))
    subprocess.check_call([nvcc()] + GENCODE + ["-shared", "-cudart", "static", "-o", SO] + objs)
    return SO


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
