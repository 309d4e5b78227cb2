"""/v1/responses requests (AIGW_SCHEMA_RESPONSES | OpenAI) through every entry point of the translate pass: the host call, the
fused small-batch kernel, the device call, the device-mapped call and the batcher.  The paths must agree with each other and
with the oracle (tests/_responses_request_oracle.py):
  * a GPU OK is an oracle OK with the same ":path", body bytes, body kind, model span and stream flag;
  * a GPU 400 is an oracle failure;
  * a GPU decline is an input the oracle fails or puts outside the restated subset (or a body over the 64 KiB class).
Corpora: tests/test_responses_request_cpu.py."""
import collections
import threading

import numpy as np
import pytest

import _responses_request_oracle as Q
import test_responses_request_cpu as G
import test_translate_edges_cpu as E
import test_translate_edges_gpu as EG

pytestmark = pytest.mark.gpu

OK, E400, DECLINED = 0, 1, 4
SCHEMA = "responses-openai"
R_TOO_LARGE = 1
CONFIGS = [("", "v1", False), ("gpt-4-turbo", "v1", False), ("", "v1", True), ("o-1", "custom/api/", False)]


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.chat_set_small_batch(-1)
    c.close()


def mapped_translate(ctx, cfg, bodies):
    """aigw_chat_translate_device_mapped: one arena, documents grouped by class through the map, one call per class"""
    import aigw_b200 as A
    n = len(bodies)
    arena, offs, lens = A.capi.pack_bodies(bodies)
    cls = np.array([E.CLASSES.index(E.class_of(len(b))) if len(b) <= E.CLASSES[-1] else len(E.CLASSES) - 1 for b in bodies])
    doc_map = np.argsort(cls, kind="stable").astype(np.uint32)
    counts = np.bincount(cls, minlength=len(E.CLASSES))
    out_cap = 2 * int(lens.astype(np.int64).sum()) + 1024 * n + 4096
    ptrs = []
    try:
        d_in, d_off, d_len, d_map = ctx.dalloc(arena.nbytes), ctx.dalloc(offs.nbytes), ctx.dalloc(lens.nbytes), ctx.dalloc(doc_map.nbytes)
        d_out, d_res, d_used = ctx.dalloc(out_cap), ctx.dalloc(n * 32), ctx.dalloc(8)
        ptrs += [d_in, d_off, d_len, d_map, d_out, d_res, d_used]
        ctx.h2d(d_in, arena); ctx.h2d(d_off, offs); ctx.h2d(d_len, lens); ctx.h2d(d_map, doc_map); ctx.memset(d_used, 0, 8)
        first = 0
        for k, c in enumerate(E.CLASSES):
            if counts[k]:
                ctx.chat_translate_device_mapped(cfg, d_in, d_off, d_len, d_map, first, int(counts[k]), c, d_out, out_cap, d_res, d_used)
                first += int(counts[k])
        res = np.zeros(n, dtype=A.DocResult); ctx.d2h(res, d_res)
        used = np.zeros(1, dtype=np.uint64); ctx.d2h(used, d_used)
        out = np.zeros(max(16, int(used[0])), dtype=np.uint8); ctx.d2h(out, d_out, int(used[0]))
    finally:
        for p in ptrs:
            ctx.dfree(p)
    return [EG.to_dict(res[i], out, bodies[i]) for i in range(n)]


def batcher_translate(ctx, cfg, bodies):
    """aigw_batcher_translate from 8 threads (the fused kernel behind it takes bodies up to the small-batch limit)"""
    b = ctx.batcher_start(cfg, max_batch=64, window_us=100)
    res = [None] * len(bodies)
    try:
        def work(t):
            for i in range(t, len(bodies), 8):
                rc, status, reason, path, body, kind = ctx.batcher_translate(b, bodies[i])
                assert rc in (0, -4), rc
                res[i] = (status, reason, path, body, kind)
        th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
        for t in th:
            t.start()
        for t in th:
            t.join()
    finally:
        ctx.batcher_stop(b)
    return res


def run_paths(ctx, bodies, override="", prefix="v1", force=False, batcher=True):
    cfg = ctx.cfg(SCHEMA, model_override=override or None, force=force, prefix=prefix)
    paths = {}
    try:
        ctx.chat_set_small_batch(0)
        paths["host"] = ctx.chat_translate(cfg, bodies)
        small = [i for i, b in enumerate(bodies) if 0 < len(b) <= E.SMALL_MAX]
        r = [None] * len(bodies)
        if small:
            ctx.chat_set_small_batch(1 << 20)
            for i, g in zip(small, ctx.chat_translate(cfg, [bodies[i] for i in small])):
                r[i] = g
        paths["fused"] = r
    finally:
        ctx.chat_set_small_batch(-1)
    groups = collections.defaultdict(list)
    for i, b in enumerate(bodies):
        groups[E.class_of(len(b)) if len(b) <= E.CLASSES[-1] else E.CLASSES[-1]].append(i)
    r = [None] * len(bodies)
    for c, idx in groups.items():
        for i, g in zip(idx, EG.device_translate(ctx, cfg, [bodies[i] for i in idx], c)):
            r[i] = g
    paths["device"] = r
    paths["mapped"] = mapped_translate(ctx, cfg, bodies)
    if batcher:
        small = [i for i, b in enumerate(bodies) if 0 < len(b) <= E.SMALL_MAX]
        r = [None] * len(bodies)
        for i, g in zip(small, batcher_translate(ctx, cfg, [bodies[i] for i in small])):
            r[i] = g
        paths["batcher"] = r
    return paths


def check(bodies, paths, override="", prefix="v1", force=False):
    """the three rules on every path, the paths equal to each other; → Counter of (status, reason) of the host call"""
    tally = collections.Counter()
    for i, body in enumerate(bodies):
        v, path, out, model, stream = Q.translate(body, override, prefix, force)
        h = paths["host"][i]
        tally[(h["status"], h["reason"])] += 1
        for name, r in paths.items():
            g = r[i]
            if g is None:
                continue
            if name == "batcher":
                assert g == (h["status"], h["reason"], h["path"], h["body"], h["body_kind"]), (name, body[:300], g, h)
                continue
            assert g == h, (name, body[:300], g, h)
        g = h
        where = (body[:400], g["status"], g["reason"], v)
        if g["status"] == OK:
            assert v == Q.OK, where
            assert g["path"].decode() == path and g["body"] == (out or b"") and g["body_kind"] == (0 if out is None else 1), (where, g, out)
            assert g["model"] == model and g["stream"] == stream, (where, g, model, stream)
        elif g["status"] == E400:
            assert v == Q.FAIL, where
        else:
            assert g["status"] == DECLINED, where
            assert v != Q.OK or (g["reason"] == R_TOO_LARGE and len(body) > E.CLASSES[-1]), where
    return tally


def report(name, tally):
    print("\n%s: OK %d, 400 %d, declined %s" % (name, sum(n for (s, _), n in tally.items() if s == OK), sum(n for (s, _), n in tally.items() if s == E400),
                                              dict(sorted(((r, n) for (s, r), n in tally.items() if s == DECLINED)))))


@pytest.mark.parametrize("override,prefix,force", CONFIGS)
def test_goldens(ctx, override, prefix, force):
    unions = [u["wrapped"].encode() for u in G.GOLD["unions"]]
    bodies = unions + [c["body"].encode() for c in G.GOLD["parse_body"]] + [c["body"].encode() for c in G.GOLD["request_body"]]
    bodies += [G.UPSTREAM[n]["requestBody"].encode() for n in ("openai - /v1/responses", "openai - /v1/responses - stream")]
    paths = run_paths(ctx, bodies, override, prefix, force)
    report("goldens %r" % ((override, prefix, force),), check(bodies, paths, override, prefix, force))
    for i, b in enumerate(bodies):   # what the oracle decodes is OK, byte-exact (checked above); outside the subset declines
        v = Q.parse_body(b)[0]
        assert (paths["host"][i]["status"] == OK) == (v == Q.OK), (b, paths["host"][i])
    for c in G.GOLD["request_body"]:
        if c["override"] == override and c["force"] == force and prefix == "v1":
            g = paths["host"][bodies.index(c["body"].encode())]
            assert g["path"] == b"/v1/responses" and g["stream"] == c.get("stream", False)


def test_other_backends_decline(ctx):
    body = b'{"model":"m","input":"hi"}'
    for base in (1, 2, 3, 4, 5, 6):
        cfg = ctx.cfg(128 | base)
        for r in ctx.chat_translate(cfg, [body]):
            assert (r["status"], r["reason"]) == (DECLINED, 19), (base, r)


@pytest.mark.parametrize("override", ["", "gpt-5-mini"])
def test_realistic_corpus(ctx, override):
    bodies = G.realistic_corpus(2000)
    paths = run_paths(ctx, bodies, override)
    tally = check(bodies, paths, override)
    report("realistic corpus (override %r)" % override, tally)
    assert tally == {(OK, 0): len(bodies)}, tally
    print("share of uncapped requests above 64 KiB: %.4f" % G.uncapped_share_above(2000))


@pytest.mark.parametrize("override", ["", "o-1"])
def test_edge_corpus(ctx, override):
    bodies = G.edge_corpus() + G.class_bound_bodies()
    tally = check(bodies, run_paths(ctx, bodies, override), override)
    report("edge corpus (override %r)" % override, tally)
    assert tally[(OK, 0)] and sum(n for (s, _), n in tally.items() if s == E400) and sum(n for (s, _), n in tally.items() if s == DECLINED)


def test_mutants(ctx):
    seeds = G.mutation_seeds()
    bodies = []
    for k, s in enumerate(seeds):
        ms = list(E.mutants(s))
        bodies += ms if len(s) < 400 else ms[k % 7::7]
    tally = check(bodies, run_paths(ctx, bodies, batcher=False))
    report("mutants (%d from %d bodies)" % (len(bodies), len(seeds)), tally)
