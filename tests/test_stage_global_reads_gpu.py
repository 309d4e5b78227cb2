"""The translate pass's index stage reads request bodies straight from global memory (chat_stage.cuh), and the emit stage stages
them by a bulk copy, or by a cooperative copy when a body is off its 16-byte alignment.  These cases put bodies where such reads can
go wrong and check every result field and record byte against the oracle, through the serial schedule and through the paired one
(index of sub-batch k+1 beside emit of sub-batch k, in a kernel of emit warps and index warps), which must agree document for
document:

  * bodies 0-15 bytes off 16-byte alignment (callers may break the alignment contract), in every size class;
  * lengths 16 / 32 / 1024 +- 1 and each class bound;
  * the last byte of the call's last body is the last byte of the device allocation that holds the bodies;
  * escapes (\\u with hex digits, \\/, odd backslash runs), a number and an escaped key spelling ("\\u006dodel") that straddle a
    lane's 32 bytes, a 1 KiB round and a 16-byte block.

The allocation-end case checks the bytes of the tail, not the absence of an over-read: cudaMalloc rounds allocations up, so a
load past the last byte reads mapped memory and neither faults nor changes an output.  That no load leaves [body, body + len)
rests on the page rule of the loaders (ldg_block_of, lookup_id<true>, hex4_at<kBodyGlobal>: only blocks or words that hold a
body byte are read); a memory checker that knows the requested size is what would catch a violation."""
import numpy as np
import pytest

import test_translate_edges_cpu as E
from test_bench_paths_gpu import OK, check_layout
from test_paired_schedule_gpu import PAIR_SUB, both_schedules
from test_translate_edges_gpu import check_contract

pytestmark = pytest.mark.gpu
SCHEMA = "aws-bedrock"
PAIR_CLASSES = (2048, 5120, 9216, 17408)   # chat_kernel.cu pair_emit_warps: the classes the paired schedule runs


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def tiny(n):
    """a JSON body of exactly n >= 13 bytes too short for the template (the oracle decides its status)"""
    if n >= 28:
        return b'{"model":"m","messages":[' + b" " * (n - 27) + b"]}"
    return b'{"model":"m"' + b" " * (n - 13) + b"}"


def common_bodies():
    """edge lengths and boundary-straddling features; every one is at most 2048 bytes, so each class's call carries them"""
    out = [tiny(n) for n in (15, 16, 17, 31, 32, 33)]
    out += [E.pad_to(E.TEMPLATES[SCHEMA], n) for n in (1023, 1024, 1025)]
    for bnd in (512, 1024):
        for f in ("esc_slash", "u_e9", "surrogate", "bs3_quote", "bs5_quote", "bs2_close", "esc_key", "number"):
            for at in range(bnd - 18, bnd + 19):
                out.append(E.straddle_body(f, at, 1300))
    return out


def class_bodies(c):
    """lengths inside class c: its lower edge, middle and upper bound, the bound last"""
    lo = E.PREV[c] + 1
    lens = [max(lo, 200), (lo + c) // 2, c - 16, c - 1]
    return [E.pad_to(E.TEMPLATES[SCHEMA], n) for n in lens]


def place(bodies, shifts):
    """one arena holding body i at an address shifts[i] bytes past a 16-byte boundary; the arena ends with the last body's last byte"""
    offs = np.zeros(len(bodies) + 1, dtype=np.uint64)
    p = 0
    for i, b in enumerate(bodies):
        p = (p + 15) // 16 * 16 + shifts[i]
        offs[i] = p
        p += len(b)
    offs[-1] = p
    arena = np.full(p, 0x20, dtype=np.uint8)
    for i, b in enumerate(bodies):
        arena[int(offs[i]):int(offs[i]) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    lens = np.fromiter((len(b) for b in bodies), dtype=np.uint32, count=len(bodies))
    return arena, offs, lens


def corpus(c):
    """every shift 0-15 for each class body, the common bodies at rotating shifts, and a body of exactly c bytes at the end"""
    bodies, shifts = [], []
    for b in class_bodies(c):
        for s in range(16):
            bodies.append(b); shifts.append(s)
    for k, b in enumerate(common_bodies()):
        bodies.append(b); shifts.append(k % 16)
    bodies.append(E.pad_to(E.TEMPLATES[SCHEMA], c)); shifts.append(7)
    return bodies, shifts


def check_oracle(bodies, recs, idx=None):
    for k, i in enumerate(idx if idx is not None else range(len(bodies))):
        b = bodies[k]
        st, reason, rec, moff, mlen, flags, kind = recs[i]
        o = E.oracle(SCHEMA, b)
        pl = len(o.path.encode()) if st == OK else 0
        g = {"status": st, "reason": reason, "path": rec[:pl], "body": rec[pl:], "model": b[moff:moff + mlen], "stream": bool(flags & 1), "body_kind": kind}
        check_contract(SCHEMA, b, g, o, i)
        if len(b) >= 200:   # the template's bodies translate: nothing here is a capacity decline
            assert st == OK, (i, len(b), st, reason)


@pytest.mark.parametrize("cls", E.CLASSES)
def test_serial_schedule(ctx, cls):
    bodies, shifts = corpus(cls)
    arena, offs, lens = place(bodies, shifts)
    assert int(offs[-2]) + int(lens[-1]) == arena.nbytes and int(lens.max()) == cls
    default, profiled = both_schedules(ctx, ctx.cfg(SCHEMA), arena, offs, lens)
    for recs, res, launches in (default, profiled):
        assert launches == 4, launches   # one serial sub-batch: index, sort, walk, emit
        check_layout(res)
    assert default[0] == profiled[0]
    check_oracle(bodies, default[0])


@pytest.mark.parametrize("cls", PAIR_CLASSES)
def test_paired_schedule(ctx, cls):
    """the corpus at the head and the tail of a call of two full sub-batches, so that its documents are indexed and emitted both by
    the stand-alone kernels and by the paired one; the documents between them share one short body"""
    bodies, shifts = corpus(cls)
    filler = E.pad_to(E.TEMPLATES[SCHEMA], 300)
    arena, offs, lens = place([filler] + bodies, [3] + shifts)
    m = len(bodies)
    n = 2 * PAIR_SUB + 2 * m
    doc = np.zeros(n, dtype=np.int64)
    doc[:m] = np.arange(1, m + 1); doc[n - m:] = np.arange(1, m + 1)
    d_offs = np.zeros(n + 1, dtype=np.uint64); d_offs[:n] = offs[doc]; d_offs[n] = offs[-1]
    d_lens = lens[doc].copy()
    paired, serial = both_schedules(ctx, ctx.cfg(SCHEMA), arena, d_offs, d_lens)
    recs, res, launches = paired
    assert launches % 3 == 1 and launches >= 7, launches
    assert (res["status"] != 255).all()
    check_layout(res)
    bad = [i for i in range(n) if recs[i] != serial[0][i]]
    assert not bad, (len(bad), bad[:10])
    check_oracle(bodies, recs, range(m))
    check_oracle(bodies, recs, range(n - m, n))
    assert all(r == recs[m] for r in recs[m:n - m:4099])

