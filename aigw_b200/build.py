"""Build libaigw_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libaigw_b200.so")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
# Per-unit ptxas flags.  ptxas -O2 / -O3 of CUDA 12.9 (V12.9.86) miscompiles the straddling-chunk loop of emit_doc
# (chat_stage.cuh) in the fused group-11 kernel.  The PTX is right: `add.s32 %k, %k, 1; … ld.shared.u32 [4*%k + s + 13632]`
# reloads s_ops[k] after ++k.  The -O3 SASS increments k and then loads 4 bytes further:
#     VIADD R23, R23, 0x1 ; IMAD R30, R23, 0x4, R20 ; LDS R26, [R30+0x3544]     (s_ops is at +0x3540: this is s_ops[k + 1])
# so every chunk that spans two copy ops skips the second one.  At -O1 the reload is `LDS [R+0x3540]` and the bytes match the
# oracle.  No other fused kernel (groups 0-10, built at -O3) contains the +0x3544 reload.  Cost of -O1 on this kernel: DESIGN.md §4.1.
# The group-12 fused kernel (Cohere /v2/rerank) shares emit_doc and gets the same faulty reload at -O3:
#     VIADD R23, R23, 0x1 ; ISETP.GE.U32.AND P2, PT, R23, R4, PT ; … IMAD R30, R23, 0x4, R20 ; LDS R26, [R30+0x3544]
# so it is built at -O1 too.
# chat_large_kernel.cu's emit has a straddling-chunk loop of its own (op ends in shared memory, advanced with ++kk); its -O3 SASS
# reloads op_end[kk], op_src[kk] and op_kind[kk] at the advanced index, so it stays at -O3.  responses_large_kernel.cu runs the same
# emit (large_request.cuh), and its -O3 SASS makes the same op-table loads (op_end +0x308 / +0x30c, op_src, op_kind), so it stays at -O3 too.
# completions_large_kernel.cu runs that emit as well and stays at -O3 for the same reason.  chat_bedrock_large_kernel.cu has an emit
# of its own (chat_large_record_impl.cuh): its straddling-chunk loop reloads a whole 16-byte op (kind, source, length, end) from
# global memory after ++k.  chat_anthropic_large_kernel.cu runs that emit too, and its -O3 SASS reloads ops[k], not ops[k + 1]:
#     VIADD R21, R21, 0x1 ; IMAD.WIDE.U32 R8, R21, 0x10, R52 ; LD.E.128 R8, desc[UR8][R8.64]     (R52: the ops base, offset +0)
# so it stays at -O3 as well.  chat_gemini_large_kernel.cu runs that emit too, and its -O3 SASS also reloads ops[k]:
#     VIADD R21, R21, 0x1 ; IMAD.WIDE.U32 R2, R21, 0x10, R48 ; LD.E.128 R8, desc[UR8][R2.64]     (R48: the ops base, offset +0)
# so it stays at -O3.  messages_large_kernel.cu runs that emit too, and its -O3 SASS also reloads ops[k]:
#     VIADD R21, R21, 0x1 ; IMAD.WIDE.U32 R2, R21, 0x10, R52 ; LD.E.128 R8, desc[UR8][R2.64]     (R52: the ops base, offset +0)
# so it stays at -O3.
PTXAS = {"chat_small_g11.cu": ["-Xptxas", "-O1"], "chat_small_g12.cu": ["-Xptxas", "-O1"]}
SOURCES = ["lib.cu", "chat_kernel.cu", "chat_walk.cu", "chat_walk_g0.cu", "chat_walk_g1.cu", "chat_walk_g2.cu", "chat_walk_g3.cu", "chat_walk_g4.cu", "chat_walk_g5.cu", "chat_walk_g6.cu", "chat_walk_g7.cu", "chat_walk_g8.cu", "chat_walk_g9.cu", "chat_walk_g10.cu", "chat_walk_g11.cu", "chat_walk_g12.cu", "chat_small_g0.cu", "chat_small_g1.cu", "chat_small_g2.cu", "chat_small_g3.cu", "chat_small_g4.cu", "chat_small_g5.cu", "chat_small_g6.cu", "chat_small_g7.cu", "chat_small_g8.cu", "chat_small_g9.cu", "chat_small_g10.cu", "chat_small_g11.cu", "chat_small_g12.cu", "sse_kernel.cu", "bedrock_stream_kernel.cu", "stream_kernel.cu", "bpe_kernel.cu", "emb_kernel.cu", "rerank_large_kernel.cu", "emb_large_kernel.cu", "chat_large_kernel.cu", "chat_large_record.cu", "chat_bedrock_large_kernel.cu", "chat_anthropic_large_kernel.cu", "chat_gemini_large_kernel.cu", "messages_large_kernel.cu", "responses_large_kernel.cu", "completions_large_kernel.cu", "mutate_kernel.cu", "batcher.cu", "sha256_kernel.cu", "cel_kernel.cu"]


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
            cmd = base + PTXAS.get(src, []) + ["-c", path, "-o", obj]
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
