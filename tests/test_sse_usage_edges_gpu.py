"""sse_usage_kernel at its chunk, group, tile, line, candidate and carry edges.  Streams are built only from line shapes the
kernel decodes (OpenAI chunks, `data: [DONE]`, comments, `event: ping`, broken JSON), so a stream's status must be exactly
test_sse_usage_edges_cpu.expected_declined, and an OK must give the oracle's usage and model bytes.  Every stream goes through
aigw_sse_usage_device from a hand-built buffer (the host form may restage the bytes) at start offsets 0-15, in one chunk, in
1-byte chunks when it is short, and cut at the tile edges of its schedule.  The generators live in
test_sse_usage_edges_cpu.py, which checks them without a GPU."""
import random

import numpy as np
import pytest

import _oracle as O
import test_sse_usage_edges_cpu as E

pytestmark = pytest.mark.gpu
DECLINED = 4


@pytest.fixture(scope="module")
def gw():
    from aigw_b200 import capi
    g = capi.Context(0)
    yield g
    g.close()


def oracle(chunks):
    s = O.SSEStream()
    acc = [-1] * 6
    for ch in chunks:
        u = s.feed(ch).as_tuple()
        acc = [n if n >= 0 else a for a, n in zip(acc, u)]
    return tuple(acc), s.model()


def run_device(gw, streams, starts):
    """streams: lists of chunks; stream i starts at an address = starts[i] (mod 16).  A padding stream of under 16 bytes without a
    newline (or of no chunks) sits in front of each, so the streams are consecutive in one buffer.  -> [(status, usage, model)]"""
    from aigw_b200 import capi
    buf, coff, cfirst, idx = bytearray(), [0], [0], []

    def add(chunks):
        for ch in chunks:
            buf.extend(ch); coff.append(len(buf))
        cfirst.append(len(coff) - 1)
    for chunks, st in zip(streams, starts):
        p = (st - len(buf)) % 16
        add([b"\x7f" * p] if p else [])
        idx.append(len(cfirst) - 1)
        add(chunks)
    n = len(cfirst) - 1
    arr = np.frombuffer(bytes(buf) + b"\0" * 64, dtype=np.uint8).copy()
    co = np.asarray(coff, dtype=np.uint64); cf = np.asarray(cfirst, dtype=np.uint32)
    d_b = gw.dalloc(len(arr)); d_o = gw.dalloc(co.nbytes); d_f = gw.dalloc(cf.nbytes); d_r = gw.dalloc(n * capi.SseResult.itemsize)
    try:
        gw.h2d(d_b, arr); gw.h2d(d_o, co); gw.h2d(d_f, cf)
        gw.memset(d_r, 0xEE, n * capi.SseResult.itemsize)
        gw.sse_usage_device(d_b, d_o, d_f, n, d_r)
        gw.sync()
        res = np.zeros(n, dtype=capi.SseResult); gw.d2h(res, d_r)
    finally:
        for p in (d_b, d_o, d_f, d_r):
            gw.dfree(p)
    out = []
    for i in idx:
        r = res[i]; m = int(r["mask"])
        tup = (int(r["input"]) if m & 1 else -1, int(r["cached"]) if m & 8 else -1, int(r["cache_creation"]) if m & 16 else -1,
               int(r["output"]) if m & 2 else -1, int(r["total"]) if m & 4 else -1, int(r["reasoning"]) if m & 32 else -1)
        out.append((int(r["status"]), tup, bytes(buf[int(r["model_off"]):int(r["model_off"]) + int(r["model_len"])])))
    real = set(idx)
    for i in range(n):
        if i not in real:
            assert int(res[i]["status"]) == 0 and int(res[i]["mask"]) == 0 and int(res[i]["model_len"]) == 0
    return out


def chunkings(s: bytes, start: int, one_byte_below=20000):
    """one chunk; 1-byte chunks for short streams; cuts at the start and end of every tile of the schedule"""
    out = [[s]]
    if len(s) < one_byte_below:
        out.append([s[i:i + 1] for i in range(len(s))])
    tiles, _ = E.tile_schedule(s, start)
    cuts = sorted({c for tb, t0, filled, *_r in tiles for c in (tb, tb + filled) if 0 < c < len(s)})
    if cuts:
        out.append([s[a:b] for a, b in zip([0] + cuts, cuts + [len(s)])])
    return out


def check(gw, items, min_ok=1):
    """items: (stream bytes, start, chunks).  Exact status, usage and model for each."""
    got = run_device(gw, [c for _s, _st, c in items], [st for _s, st, _c in items])
    n_ok = 0
    for (s, st, chunks), (status, tup, model) in zip(items, got):
        want_decl = E.expected_declined(s)
        assert status == (DECLINED if want_decl else 0), (len(s), st, s[:200], status)
        if status == 0:
            eu, em = oracle(chunks)
            assert (tup, model) == (eu, em), (len(s), st, len(chunks), tup, eu, model, em)
            n_ok += 1
    assert n_ok >= min_ok
    return n_ok


def expand(streams, starts=range(16), one_byte_below=20000):
    return [(s, st, ch) for s in streams for st in starts for ch in chunkings(s, st, one_byte_below)]


def test_usage_found_only_through_next_u(gw):
    items = []
    for st in range(16):
        for kw in ({}, {"modulus": E.GROUP, "addr": 511}, {"modulus": E.GROUP, "addr": 0}):
            s = E.s_next_u(st, **kw)
            items += [(s, st, ch) for ch in chunkings(s, st)]
    check(gw, items, min_ok=len(items))
    for s, st, ch in items[:3]:
        assert oracle(ch)[0][0] == 11       # the usage comes from that line


def test_model_found_only_by_the_walk_all_pass(gw):
    items = expand(E.s_second_pass(0))
    check(gw, items, min_ok=len(items))


def test_tile_boundaries(gw):
    streams = [s for _n, s in E.boundary_streams()]
    items = expand(streams, starts=range(16), one_byte_below=12000)
    check(gw, items, min_ok=len(items) // 2)
    names = dict(E.boundary_streams())
    got = run_device(gw, [[names[k]] for k in ("lines_512", "lines_513", "line_8192", "line_8193", "tail_8192", "tail_8193", "cand_64", "cand_65")], [0] * 8)
    assert [g[0] for g in got] == [0, DECLINED, 0, DECLINED, 0, DECLINED, 0, 0]


def test_usage_key_split_by_the_tile_end(gw):
    items = expand(E.usage_split_stream(), starts=range(16), one_byte_below=0)
    check(gw, items, min_ok=len(items))
    assert all(oracle(ch)[0][0] == 6 for _s, _st, ch in items)


@pytest.mark.parametrize("mb,seed", [(1, 1), (4, 2)])
def test_megabyte_streams(gw, mb, seed):
    s = E.big_stream(mb, seed)
    items = [(s, st, ch) for st in (0, 7, 15) for ch in chunkings(s, st, one_byte_below=0)]
    r = random.Random(seed)
    cuts = sorted(r.sample(range(1, len(s)), 300))
    items.append((s, 3, [s[a:b] for a, b in zip([0] + cuts, cuts + [len(s)])]))
    check(gw, items, min_ok=len(items))


def test_thousands_of_mixed_streams(gw):
    r = random.Random(11)
    pool = [s for _n, s in E.boundary_streams()] + E.s_second_pass(0) + E.usage_split_stream() + [E.s_next_u(st) for st in range(16)]
    pool += [E.chunk("a") + E.DONE, E.COMMENT, b"data: {oops", b"", b"\n" * 513, b"\n" * 512]
    items = []
    for _ in range(3000):
        x = r.random()
        if x < 0.05:
            items.append((b"", r.randrange(16), []))                     # a stream of no chunks
        elif x < 0.1:
            items.append((b"", r.randrange(16), [b""]))                  # one empty chunk
        else:
            s = r.choice(pool)
            k = r.randint(0, 5)
            cuts = sorted(r.sample(range(1, len(s)), min(k, max(0, len(s) - 1)))) if len(s) > 1 else []
            items.append((s, r.randrange(16), [s[a:b] for a, b in zip([0] + cuts, cuts + [len(s)])]))
    n_ok = check(gw, items, min_ok=1000)
    assert sum(1 for s, _st, _c in items if E.expected_declined(s)) >= 200 and n_ok >= 2000
