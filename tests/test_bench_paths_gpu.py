"""The schedules bench.py and tools/bench_zipf.py measure, run at the sizes where they change shape: a device call across translate
sub-batches, a host call across 256 MiB chunks and their three reused slots, the class-mapped device call, the stream calls'
three input feeds with the stream pool grown under live streams, and the device twins of the host calls of bench configs 3-5.
Every call is checked against a call that does not take the schedule under test, per document, and a sample against the oracle."""
import ctypes as C
import json
import random
import types

import numpy as np
import pytest

import _oracle as O
import _responses_oracle as R
import _workload as W
import test_embeddings_count_gpu as TE
import test_responses_gpu as TR
import test_stream_gpu as TS

pytestmark = pytest.mark.gpu
OK = 0
SUB_BATCH = 262144        # documents per sub-batch of a device call (chat_kernel.cu), below the workspace cap
CHUNK = 256 << 20         # bytes per pipeline chunk of the host call (lib.cu)


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def records(res, out):
    """per document: (status, reason, record bytes or b"", model span, flags, body kind)"""
    r = []
    for x in res:
        st = int(x["status"])
        o = int(x["out_off"]); n = int(x["path_len"]) + int(x["body_len"])
        r.append((st, int(x["reason"]), bytes(out[o:o + n]) if st == OK else b"", int(x["model_off"]), int(x["model_len"]), int(x["flags"]), int(x["body_kind"])))
    return r


class DeviceCorpus:
    """a corpus in device memory with the output arena and result table of one device call; free() releases all of it"""

    def __init__(self, ctx, arena, offs, lens, out_cap=None):
        self.ctx, self.n = ctx, len(lens)
        self.out_cap = out_cap or int(arena.nbytes * 1.25) + self.n * 600 + 4096
        self.ptrs = []
        try:
            self.d_in = self._alloc(arena.nbytes); self.d_off = self._alloc(offs.nbytes); self.d_len = self._alloc(lens.nbytes)
            self.d_out = self._alloc(self.out_cap); self.d_res = self._alloc(self.n * 32); self.d_used = self._alloc(8)
            ctx.h2d(self.d_in, arena); ctx.h2d(self.d_off, offs); ctx.h2d(self.d_len, lens)
        except BaseException:
            self.free()
            raise

    def _alloc(self, n):
        p = self.ctx.dalloc(n)
        self.ptrs.append(p)
        return p

    def reset(self):
        self.ctx.memset(self.d_used, 0, 8)
        self.ctx.memset(self.d_res, 0xff, self.n * 32)   # a document the call never reaches keeps status 255

    def fetch(self):
        import aigw_b200 as A
        res = np.zeros(self.n, dtype=A.DocResult); self.ctx.d2h(res, self.d_res)
        used = np.zeros(1, dtype=np.uint64); self.ctx.d2h(used, self.d_used)
        out = np.zeros(max(16, int(used[0])), dtype=np.uint8); self.ctx.d2h(out, self.d_out, int(used[0]))
        return res, out

    def free(self):
        for p in self.ptrs:
            self.ctx.dfree(p)
        self.ptrs = []


def check_layout(res):
    """records are 16-byte aligned and do not overlap"""
    ok = res["status"] == OK
    o = res["out_off"][ok].astype(np.int64); l = res["path_len"][ok].astype(np.int64) + res["body_len"][ok].astype(np.int64)
    order = np.argsort(o); o, l = o[order], l[order]
    assert (o % 16 == 0).all() and (o[1:] >= o[:-1] + l[:-1]).all()


def check_oracle(schema, arena, offs, lens, recs, idx):
    for i in idx:
        b = bytes(arena[int(offs[i]):int(offs[i]) + int(lens[i])])
        t = O.chat_translate(schema, b)
        st, _, rec, *_ = recs[i]
        assert st == OK and t.status == O.OK, (i, st, t.err)
        pl = len(t.path.encode())
        assert rec[:pl].decode() == t.path and rec[pl:] == (t.body if t.body_kind == O.BYTES else b""), i


# ---------------------------------------------------------------- B1: device call across sub-batches
def test_device_call_across_sub_batches(ctx):
    n = SUB_BATCH + 4097
    arena, offs, lens = W.chat_corpus(2, 0, n, target=1024)
    assert int(lens.max()) <= 2048
    cfg = ctx.cfg("aws-bedrock")
    dc = DeviceCorpus(ctx, arena, offs, lens)
    try:
        dc.reset()
        ctx.chat_translate_device(cfg, dc.d_in, dc.d_off, dc.d_len, n, int(lens.max()), dc.d_out, dc.out_cap, dc.d_res, dc.d_used)
        launches = ctx.chat_last_profile()["launches"]
        res, out = dc.fetch()
        # the serial pass the bench times per stage: one stream, the stages back to back
        ctx.chat_set_profile(True)
        try:
            dc.reset()
            ctx.chat_translate_device(cfg, dc.d_in, dc.d_off, dc.d_len, n, int(lens.max()), dc.d_out, dc.out_cap, dc.d_res, dc.d_used)
            prof = ctx.chat_last_profile()
        finally:
            ctx.chat_set_profile(False)
        res2, out2 = dc.fetch()
    finally:
        dc.free()
    print("device call of", n, "bodies: launches", launches, "profiled launches", prof["launches"])
    assert launches >= 8 and prof["launches"] >= 8
    assert (res["status"] == OK).all(), np.unique(res["status"], return_counts=True)
    check_layout(res)
    recs = records(res, out)
    assert recs == records(res2, out2)
    idx = sorted(set(range(SUB_BATCH - 2048, min(n, SUB_BATCH + 2048))) | set(range(0, n, 64)))
    check_oracle("aws-bedrock", arena, offs, lens, recs, idx)


def test_device_call_splits_under_workspace_cap(ctx):
    """the 65536 class needs 67 232 bytes of workspace per document: 60 000 documents do not fit the workspace (3 GiB plus the
    allocator's eighth of headroom) and run in two sub-batches.  The workspace depends on the class, not on the body lengths, so most
    bodies are small (the class is the call's max_len) and device memory stays low; one in 100, spread over both sub-batches, is a
    34-40 KB body."""
    n = 60000
    small = W.chat_corpus(7, 0, n, target=1024)
    big = W.chat_corpus(7, 10_000_000, n // 100, target=37000, jitter=3000)
    bodies = []
    for i in range(n):
        (a, o, l), j = (big, i // 100) if i % 100 == 50 else (small, i)
        bodies.append(bytes(a[int(o[j]):int(o[j]) + int(l[j])]))
    import aigw_b200 as A
    arena, offs, lens = A.capi.pack_bodies(bodies)
    assert int(lens.max()) > 33792
    cfg = ctx.cfg("aws-bedrock")
    dc = DeviceCorpus(ctx, arena, offs, lens)
    try:
        dc.reset()
        ctx.chat_translate_device(cfg, dc.d_in, dc.d_off, dc.d_len, n, int(lens.max()), dc.d_out, dc.out_cap, dc.d_res, dc.d_used)
        launches = ctx.chat_last_profile()["launches"]
        res, out = dc.fetch()
    finally:
        dc.free()
    print("65536-class device call of", n, "bodies: launches", launches)
    assert launches >= 8
    assert (res["status"] == OK).all()
    check_layout(res)
    recs = records(res, out)
    # the host call buckets the same documents by class into one launch sequence per class
    hres, hout, _ = ctx.chat_translate_host(cfg, arena, offs[:n], lens)
    assert recs == records(hres, hout)
    check_oracle("aws-bedrock", arena, offs, lens, recs, list(range(0, n, 97)) + list(range(50, n, 100)))


# ---------------------------------------------------------------- B2 / B3: host pipeline across chunks, class-mapped device calls
@pytest.fixture(scope="module")
def chunked_corpus():
    """more than three 256 MiB chunks of bodies from 1.1 to 4.9 KB: every chunk holds two size classes"""
    n = 300_000
    arena, offs, lens = W.chat_corpus(11, 0, n, target=3000, jitter=1900)
    assert int(offs[-1]) > 3 * CHUNK + CHUNK // 4
    return arena, offs, lens


def test_host_pipeline_across_chunks(ctx, chunked_corpus):
    arena, offs, lens = chunked_corpus
    n = len(lens)
    cfg = ctx.cfg("aws-bedrock")
    res, out, stats = ctx.chat_translate_host(cfg, arena, offs[:n], lens)
    host = records(res, out)
    check_layout(res)
    chunks = -(-int(offs[-1]) // CHUNK)
    print("host call:", n, "bodies,", int(offs[-1]) >> 20, "MiB,", stats["gpu_launches"], "launches")
    # every chunk runs two classes (4 launches each) over its document map
    assert stats["gpu_launches"] >= chunks * 2 * 4 and chunks >= 4
    dc = DeviceCorpus(ctx, arena, offs, lens)
    try:
        dc.reset()
        ctx.chat_translate_device(cfg, dc.d_in, dc.d_off, dc.d_len, n, int(lens.max()), dc.d_out, dc.out_cap, dc.d_res, dc.d_used)
        dres, dout = dc.fetch()
    finally:
        dc.free()
    dev = records(dres, dout)
    assert sum(1 for r in host if r[0] == OK) == n
    assert host == dev
    check_oracle("aws-bedrock", arena, offs, lens, host, range(0, n, 499))


def test_device_mapped_by_class(ctx, chunked_corpus):
    """aigw_chat_translate_device_mapped as tools/bench_zipf.py calls it: documents grouped by class, one call per class"""
    import aigw_b200 as A
    arena, offs, lens = chunked_corpus
    n = len(lens)
    cfg = ctx.cfg("aws-bedrock")
    cls = np.searchsorted(np.array([2048, 5120, 9216, 17408, 33792, 65536]), lens)
    doc_map = np.argsort(cls, kind="stable").astype(np.uint32)
    counts = np.bincount(cls, minlength=6)
    assert (counts > 0).sum() == 2
    dc = DeviceCorpus(ctx, arena, offs, lens)
    try:
        d_map = dc._alloc(doc_map.nbytes); ctx.h2d(d_map, doc_map)
        dc.reset()
        first = 0
        for k, c in enumerate((2048, 5120, 9216, 17408, 33792, 65536)):
            if counts[k]:
                ctx.chat_translate_device_mapped(cfg, dc.d_in, dc.d_off, dc.d_len, d_map, first, int(counts[k]), c, dc.d_out, dc.out_cap, dc.d_res, dc.d_used)
                first += int(counts[k])
        mres, mout = dc.fetch()
    finally:
        dc.free()
    check_layout(mres)
    res, out, _ = ctx.chat_translate_host(cfg, arena, offs[:n], lens)
    assert records(mres, mout) == records(res, out)


# ---------------------------------------------------------------- B4: stream calls, three input feeds
def soa_dicts(res, arena):
    out = []
    for r in res:
        tot = int(r["out_len"]) + int(r["model_len"])
        raw = C.string_at(arena + int(r["out_off"]), tot) if tot else b""
        m = int(r["mask"])
        usage = (int(r["input"]) if m & 1 else -1, int(r["cached"]) if m & 8 else -1, int(r["cache_creation"]) if m & 16 else -1,
                 int(r["output"]) if m & 2 else -1, int(r["total"]) if m & 4 else -1, int(r["reasoning"]) if m & 32 else -1)
        out.append({"status": int(r["status"]), "body_kind": int(r["body_kind"]), "reason": int(r["reason"]), "body": raw[:int(r["out_len"])], "model": raw[int(r["out_len"]):],
                    "usage": usage, "carry_len": int(r["carry_len"])})
    return out


def _cut(rng, data, k):
    cuts = sorted(rng.sample(range(1, len(data)), min(k, len(data) - 1)))
    return [data[a:b] for a, b in zip([0] + cuts, cuts + [len(data)])]


def stream_corpus(kind, n, seed):
    """n streams of one kind, each a list of chunks; eos on the last chunk where the kind flushes at end of stream"""
    rng = random.Random(seed)
    if kind == "openai":
        buf, coff, cfirst = W.sse_corpus(seed, 0, n, chunks=24)
        raw = bytes(buf)
        return [_cut(rng, raw[int(coff[int(cfirst[s])]):int(coff[int(cfirst[s + 1])])], rng.randint(1, 11)) for s in range(n)]
    if kind == "aws-bedrock":
        _, _, streams = W.bedrock_stream_corpus(n, seed=seed)
        return [_cut(rng, d, rng.randint(1, 9)) for d in streams]
    if kind == "gcp-anthropicai":
        out = []
        for _ in range(n):
            ev = ["start", "text_start"] + ["text"] * rng.randint(1, 6) + ["block_stop", "tool_start", "tool_delta", "block_stop", "delta", "stop"]
            data = "".join(TS._an_event(rng, k) + "\n\n" for k in ev).encode()
            out.append(_cut(rng, data, rng.randint(0, 12)))
        return out
    if kind == "openai-responses":
        return [TR._chunk(rng, TR._stream(rng, True)) for _ in range(n)]
    raise KeyError(kind)


STREAM_OPEN = {"openai": (b"req-model", b"", 0), "aws-bedrock": (b"model-x", b"req-1", 1700000000), "gcp-anthropicai": (b"claude-x", b"", 99), "openai-responses": (b"req-model", b"", 0)}
EOS_KINDS = ("aws-bedrock", "gcp-anthropicai")


class Oracle:
    def __init__(self, kind):
        self.kind = kind
        m, rid, created = STREAM_OPEN[kind]
        self.s = {"openai": lambda: O.SSEStream(), "aws-bedrock": lambda: O.BedrockStream(m, rid, created), "gcp-anthropicai": lambda: O.AnthropicStream(m, created),
                  "openai-responses": lambda: R.ResponsesSSEStream(m)}[kind]()
        self.dead = False

    def check(self, chunk, eos, g):
        if self.dead:
            return
        if self.kind == "openai":
            u = self.s.feed(chunk)
            assert g["status"] == OK and g["usage"] == u.as_tuple() and g["carry_len"] == self.s.buffered()
            assert g["model"] == (self.s.model() or b"req-model")
        elif self.kind == "aws-bedrock":
            o, u = self.s.feed(chunk, eos)
            assert g["status"] == OK and g["body"] == o and g["usage"] == u.as_tuple()
        elif self.kind == "gcp-anthropicai":
            s, o, u = self.s.feed(chunk, eos)
            assert g["status"] == s
            if s == OK:
                assert g["body"] == o and g["usage"] == u.as_tuple()
            else:
                self.dead = True
        else:
            v, u = self.s.feed(chunk)
            if v == R.OUT:
                self.dead = True
                return
            assert g["status"] == OK and g["usage"] == u.as_tuple() and g["model"] == self.s.model()


def feed_three_ways(ctx, kind, streams, pinned):
    """one round per chunk index: the same chunks through a pinned base (unaligned offsets, read in place), a pageable numpy base
    (staged), and aigw_stream_chunks; the three must agree, and the per-call results are returned once"""
    n = len(streams)
    m, rid, created = STREAM_OPEN[kind]
    hs = [np.array(ctx.stream_open(kind, m, rid, created, n=n), dtype=np.uint64) for _ in range(3)]
    rng = random.Random(5)
    got = []
    orc = [Oracle(kind) for _ in range(n)]
    try:
        for rnd in range(max(len(s) for s in streams)):
            idx = [i for i in range(n) if rnd < len(streams[i])]
            chunks = [streams[i][rnd] for i in idx]
            eos = np.array([kind in EOS_KINDS and rnd == len(streams[i]) - 1 for i in idx], dtype=np.uint8)
            offs = np.zeros(len(idx), dtype=np.uint64); lens = np.array([len(c) for c in chunks], dtype=np.uint32)
            pos = 1
            for k, ch in enumerate(chunks):
                offs[k] = pos
                pinned[pos:pos + len(ch)] = np.frombuffer(ch, dtype=np.uint8)
                pos += len(ch) + rng.randint(1, 15)   # chunk starts deliberately not 16-byte aligned
                if pos % 16 == 0:
                    pos += 1
            assert pos < len(pinned)
            pageable = np.array(pinned[:pos])
            res, arena = ctx.stream_chunks_soa(hs[0][idx], pinned, offs, lens, eos)
            a = soa_dicts(res, arena)
            res, arena = ctx.stream_chunks_soa(hs[1][idx], pageable, offs, lens, eos)
            b = soa_dicts(res, arena)
            c = ctx.stream_chunks([int(h) for h in hs[2][idx]], chunks, list(eos))
            assert a == b == c, (kind, rnd)
            for i, ch, e, g in zip(idx, chunks, eos, c):
                orc[i].check(ch, bool(e), g)
            got += a
    finally:
        for h in hs:
            ctx.stream_close(h)
    return got


@pytest.mark.parametrize("kind", ["openai", "aws-bedrock", "gcp-anthropicai", "openai-responses"])
def test_stream_chunks_soa_feeds(ctx, kind):
    streams = stream_corpus(kind, 96, seed=4)
    size = 64 + sum(max(len(c) for c in s) + 32 for s in streams)
    pinned, pp = ctx.host_array(size)
    try:
        res = feed_three_ways(ctx, kind, streams, pinned)
    finally:
        ctx.host_free(pp)
    assert sum(1 for r in res if r["status"] == OK) > len(res) * 0.8


def test_stream_pool_growth_under_live_streams():
    """1000 streams fed halfway, 4000 more opened (the pool grows past 1024 slots and copies the live ones), then all finished: the
    first 1000 give what an uninterrupted run gives.  A closed handle is refused; a reused slot starts clean."""
    import aigw_b200 as A
    streams = stream_corpus("aws-bedrock", 1000, seed=9)
    rounds = max(len(s) for s in streams)

    def run(ctx, grow):
        hs = ctx.stream_open("aws-bedrock", b"model-x", b"req-1", 1700000000, n=len(streams))
        out = [[] for _ in streams]
        extra = []
        for rnd in range(rounds):
            if grow and rnd == rounds // 2:
                extra = ctx.stream_open("aws-bedrock", b"other", b"req-2", 1, n=4000)
            idx = [i for i in range(len(streams)) if rnd < len(streams[i])]
            got = ctx.stream_chunks([hs[i] for i in idx], [streams[i][rnd] for i in idx], [rnd == len(streams[i]) - 1 for i in idx])
            for i, g in zip(idx, got):
                out[i].append(g)
        return hs, extra, out

    c1 = A.Context(0)
    try:
        _, _, plain = run(c1, False)
    finally:
        c1.close()
    c2 = A.Context(0)
    try:
        hs, extra, grown = run(c2, True)
        assert len(extra) == 4000
        assert grown == plain
        # the finished streams give what the oracle gives
        for i in range(0, len(streams), 50):
            ref, _ = O.bedrock_stream(b"".join(streams[i]), None, b"model-x", b"req-1", 1700000000)
            assert b"".join(g["body"] for g in grown[i]) == ref
        # a closed handle is refused, and a reused slot starts clean
        assert c2.stream_close(hs[:10]) == 0
        assert c2.stream_close(hs[:1]) == -2
        with pytest.raises(RuntimeError):
            c2.stream_chunks([hs[0]], [streams[0][0]], [False])
        again = c2.stream_open("aws-bedrock", b"model-x", b"req-1", 1700000000, n=10)
        assert {h & 0xffffffff for h in again} == {h & 0xffffffff for h in hs[:10]} and not set(again) & set(hs[:10])   # same slots, new generation
        for k in range(10):
            got = [c2.stream_chunks([again[k]], [ch], [j == len(streams[k]) - 1])[0] for j, ch in enumerate(streams[k])]
            assert got == plain[k]
        c2.stream_close(again); c2.stream_close(extra); c2.stream_close(hs[10:])
    finally:
        c2.close()


# ---------------------------------------------------------------- B5: device twins of the host calls
def test_embeddings_count_device_matches_host(ctx):
    import aigw_b200 as A
    vocab = TE.VOCAB
    bpe = ctx.bpe_load(vocab["byte_to_id"], vocab["merges"])
    r = random.Random(5)
    ws = TE.words(r)
    bodies = [TE.emb_body(r, ws) for _ in range(300)]
    bodies += [json.dumps({"model": "text-embedding-3-small", "input": [TE.text(r, ws, 64) for _ in range(1024)]}, separators=(",", ":")).encode() for _ in range(16)]
    arena, offs, lens = A.capi.pack_bodies(bodies)
    n = len(bodies)
    ptrs = []
    try:
        host, _ = ctx.embeddings_count_host(bpe, arena, offs[:n], lens)
        for p in (arena.nbytes, offs.nbytes, lens.nbytes, n * A.capi.EmbCountResult.itemsize):
            ptrs.append(ctx.dalloc(p))
        d_b, d_o, d_l, d_r = ptrs
        ctx.h2d(d_b, arena); ctx.h2d(d_o, offs); ctx.h2d(d_l, lens)
        ctx.embeddings_count_device(bpe, d_b, d_o, d_l, n, int(lens.max()), int(offs[n]), d_r)
        dev = np.zeros(n, dtype=A.capi.EmbCountResult); ctx.d2h(dev, d_r)
        # BPE counts of the same texts through the device call
        texts = [TE.text(r, ws, r.choice([0, 5, 64, 300])).encode() for _ in range(2000)]
        tarena, toffs, tlens = A.capi.pack_bodies(texts)
        hc, _ = ctx.bpe_count_host(bpe, tarena, toffs[:len(texts)], tlens)
        t_ptrs = [ctx.dalloc(x) for x in (tarena.nbytes, toffs.nbytes, tlens.nbytes, len(texts) * 4)]
        ptrs += t_ptrs
        ctx.h2d(t_ptrs[0], tarena); ctx.h2d(t_ptrs[1], toffs); ctx.h2d(t_ptrs[2], tlens)
        ctx.bpe_count_device(bpe, t_ptrs[0], t_ptrs[1], t_ptrs[2], len(texts), t_ptrs[3])
        dc = np.zeros(len(texts), dtype=np.uint32); ctx.d2h(dc, t_ptrs[3])
        # the host call against the oracle (test_embeddings_count_gpu.check reads the table from its first argument)
        ok, decl, err = TE.check(types.SimpleNamespace(bpe=bpe, embeddings_count=ctx.embeddings_count), bodies, O.Bpe(vocab))
    finally:
        for p in ptrs:
            ctx.dfree(p)
        ctx.bpe_free(bpe)
    fields = [f for f in A.capi.EmbCountResult.names if f not in ("first_text", "reserved")]   # first_text: a row of the text table, taken in arrival order
    assert (dev[fields] == host[fields]).all()
    assert (dc == hc).all() and (hc == O.Bpe(vocab).count([t.decode() for t in texts])).all()
    assert ok > n // 2


def test_bedrock_stream_and_body_mutate_device_match_host(ctx):
    import aigw_b200 as A
    buf, soff, streams = W.bedrock_stream_corpus(200, seed=8)
    hres, hout, _ = ctx.bedrock_stream_host(buf, soff, "model-x", "req-1", 1700000000)
    hrec = [(int(x["status"]), bytes(hout[int(x["out_off"]):int(x["out_off"]) + int(x["out_len"])])) for x in hres]
    n = len(streams)
    cap = 16 * len(buf) + 4096 * n
    ptrs = [ctx.dalloc(x) for x in (buf.nbytes + 64, soff.nbytes, cap, n * A.capi.StreamResult.itemsize, 8)]
    try:
        ctx.h2d(ptrs[0], buf); ctx.h2d(ptrs[1], soff); ctx.memset(ptrs[4], 0, 8)
        ctx.bedrock_stream_device(ptrs[0], ptrs[1], n, int(soff[-1]), ptrs[2], cap, ptrs[3], ptrs[4], "model-x", "req-1", 1700000000)
        dres = np.zeros(n, dtype=A.capi.StreamResult); ctx.d2h(dres, ptrs[3])
        used = np.zeros(1, dtype=np.uint64); ctx.d2h(used, ptrs[4])
        dout = np.zeros(max(16, int(used[0])), dtype=np.uint8); ctx.d2h(dout, ptrs[2], int(used[0]))
    finally:
        for p in ptrs:
            ctx.dfree(p)
    drec = [(int(x["status"]), bytes(dout[int(x["out_off"]):int(x["out_off"]) + int(x["out_len"])])) for x in dres]
    assert drec == hrec
    for i in range(0, n, 10):
        ref, _ = O.bedrock_stream(streams[i], None, b"model-x", b"req-1", 1700000000)
        assert hrec[i] == (OK, ref)
    # body mutation: the device call against the host call on the benchmark's bodies
    arena, offs, lens = W.chat_corpus(2, 0, 2000)
    removes, sets = ["stream_options"], [("temperature", "0.5"), ("max_tokens", "150"), ("custom_field", '"route-level-value"')]
    hres, hout, _ = ctx.body_mutate_host(removes, sets, arena, offs[:2000], lens)
    hrec = [(int(x["status"]), int(x["flags"]), bytes(hout[int(x["out_off"]):int(x["out_off"]) + int(x["out_len"])]) if x["status"] == OK else b"") for x in hres]
    cap = 2 * arena.nbytes + 4096
    ptrs = [ctx.dalloc(x) for x in (arena.nbytes, offs.nbytes, lens.nbytes, cap, 2000 * A.capi.MutResult.itemsize, 8)]
    try:
        ctx.h2d(ptrs[0], arena); ctx.h2d(ptrs[1], offs); ctx.h2d(ptrs[2], lens); ctx.memset(ptrs[5], 0, 8)
        ctx.body_mutate_device(removes, sets, ptrs[0], ptrs[1], ptrs[2], 2000, int(lens.max()), ptrs[3], cap, ptrs[4], ptrs[5])
        dres = np.zeros(2000, dtype=A.capi.MutResult); ctx.d2h(dres, ptrs[4])
        used = np.zeros(1, dtype=np.uint64); ctx.d2h(used, ptrs[5])
        dout = np.zeros(max(16, int(used[0])), dtype=np.uint8); ctx.d2h(dout, ptrs[3], int(used[0]))
    finally:
        for p in ptrs:
            ctx.dfree(p)
    drec = [(int(x["status"]), int(x["flags"]), bytes(dout[int(x["out_off"]):int(x["out_off"]) + int(x["out_len"])]) if x["status"] == OK else b"") for x in dres]
    assert drec == hrec
    assert sum(1 for r in hrec if r[0] == OK) > 1500
