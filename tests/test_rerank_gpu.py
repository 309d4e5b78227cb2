"""Cohere /v2/rerank on the GPU: requests (AIGW_SCHEMA_RERANK_COHERE) through every entry point of the translate pass (the host
call, the fused small-batch kernel, the device call, the device-mapped call and the batcher), buffered response usage
(aigw_rerank_response_usage_*) and the error schema (AIGW_SCHEMA_RESP_ERROR_COHERE), against the oracle (tests/_rerank_oracle.py):
  * a GPU OK is an oracle OK with the same ":path", body bytes, body kind and model span;
  * a GPU 400 (request) or AIGW_INTERNAL (response) is an oracle failure;
  * a GPU decline is an input the oracle fails or puts outside the subset, or a capacity / size decline.
Corpora: tests/test_rerank_cpu.py."""
import collections

import numpy as np
import pytest

import _rerank_oracle as Q
import test_rerank_cpu as G
import test_responses_request_gpu as RG
import test_translate_edges_cpu as E
import test_translate_edges_gpu as EG

pytestmark = pytest.mark.gpu

OK, E400, INTERNAL, DECLINED = 0, 1, 3, 4
SCHEMA = "rerank-cohere"
R_TOO_LARGE, R_TOKENS, R_SCHEMA = 1, 5, 19
CAPACITY = (R_TOKENS, 6, 7)   # tokens, ops, scratch
CONFIGS = [("", "v2", False), ("rerank-english-v3", "v2", False), ("", "v2", True), ("o-1", "/v2//beta/./x/../", True), ("", "", False)]


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.chat_set_small_batch(-1)
    c.close()


def run_paths(ctx, bodies, override="", version="v2", force=False, batcher=True):
    cfg = ctx.cfg(SCHEMA, model_override=override or None, force=force, api_version=version or None)
    paths = {}
    small = [i for i, b in enumerate(bodies) if 0 < len(b) <= E.SMALL_MAX]
    try:
        ctx.chat_set_small_batch(0)
        paths["host"] = ctx.chat_translate(cfg, bodies)
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
        groups[E.class_of(len(b))].append(i)
    r = [None] * len(bodies)
    for c, idx in groups.items():
        for i, g in zip(idx, EG.device_translate(ctx, cfg, [bodies[i] for i in idx], c)):
            r[i] = g
    paths["device"] = r
    paths["mapped"] = RG.mapped_translate(ctx, cfg, bodies)
    if batcher:
        r = [None] * len(bodies)
        for i, g in zip(small, RG.batcher_translate(ctx, cfg, [bodies[i] for i in small])):
            r[i] = dict(zip(("status", "reason", "path", "body", "body_kind"), g))
        paths["batcher"] = r
    return paths


KEYS = ("status", "reason", "path", "body", "body_kind")


def check(bodies, paths, override="", version="v2", force=False):
    """the three rules on every path, the paths equal where none declined for capacity; → Counter of (status, reason) of the host call"""
    tally = collections.Counter()
    for i, body in enumerate(bodies):
        v, path, out, model = Q.translate(body, override, version, force)
        got = {name: r[i] for name, r in paths.items() if r[i] is not None}
        tally[(got["host"]["status"], got["host"]["reason"])] += 1
        for name, g in got.items():
            where = (name, body[:300], g["status"], g["reason"], v)
            if g["status"] == OK:
                assert v == Q.OK, where
                assert g["path"].decode() == path and g["body"] == (out or b"") and g["body_kind"] == (0 if out is None else 1), (where, g, out)
                if "model" in g:
                    assert g["model"] == model and g["stream"] is False, (where, g, model)
            elif g["status"] == E400:
                assert v == Q.FAIL, where
            else:
                assert g["status"] == DECLINED, where
                assert v != Q.OK or g["reason"] in CAPACITY or (g["reason"] == R_TOO_LARGE and len(body) > E.CLASSES[-1]), where
        settled = {n: g for n, g in got.items() if not (g["status"] == DECLINED and g["reason"] in CAPACITY)}
        for name, g in settled.items():
            h = settled.get("host") or next(iter(settled.values()))
            assert all(g[k] == h[k] for k in KEYS), (name, body[:300], g, h)
    return tally


def report(name, tally):
    n = sum(tally.values())
    ok = sum(c for (s, _), c in tally.items() if s == OK)
    print("\n%s: %d bodies, OK %d (%.2f %%), 400 %d, declined by reason %s" % (
        name, n, ok, 100.0 * ok / n, sum(c for (s, _), c in tally.items() if s == E400),
        dict(sorted(((r, c) for (s, r), c in tally.items() if s == DECLINED)))))


@pytest.mark.parametrize("override,version,force", CONFIGS)
def test_goldens(ctx, override, version, force):
    bodies = [c["body"].encode() for c in G.GOLD["parse_body"]] + [G.GOLD["request_body"][0]["body"].encode()]
    paths = run_paths(ctx, bodies, override, version, force)
    report("goldens %r" % ((override, version, force),), check(bodies, paths, override, version, force))
    assert [paths["host"][i]["status"] for i in range(len(bodies))] == [E400, OK, OK]
    for c in G.GOLD["request_body"]:
        if (c["override"], c["force"], c["version"]) == (override, force, version):
            g = paths["host"][-1]
            assert g["path"].decode() == c["exp_path"] and g["model"] == b"rerank-english-v3"
            assert (c["exp_body_contains"].encode() in g["body"]) if c["exp_body_contains"] else g["body"] == (c["body"].encode() if force else b"")


def test_other_backends_decline(ctx):
    """GetTranslator serves only Cohere under the rerank family, and Cohere alone is no chat schema"""
    body = b'{"model":"m","query":"q","documents":["a"]}'
    for schema in (512, 513, 514, 515, 516, 517, 518, 519 | 256, 519 | 128, 519 | 64, 519 | 32, 7):
        for small in (0, 1 << 20):
            try:
                ctx.chat_set_small_batch(small)
                r = ctx.chat_translate(ctx.cfg(schema, api_version="v2"), [body])[0]
            finally:
                ctx.chat_set_small_batch(-1)
            assert (r["status"], r["reason"]) == (DECLINED, R_SCHEMA), (schema, small, r)


@pytest.mark.parametrize("override", ["", "rerank-v3.5"])
def test_realistic_corpus(ctx, override):
    """every realistic rerank decodes; the only declines are size or token-capacity declines, counted and reported"""
    bodies = G.realistic_corpus(2000)
    paths = run_paths(ctx, bodies, override)
    tally = check(bodies, paths, override)
    report("realistic corpus (override %r)" % override, tally)
    assert set(tally) <= {(OK, 0), (DECLINED, R_TOKENS), (DECLINED, R_TOO_LARGE)}, tally
    assert tally[(OK, 0)] >= 0.98 * len(bodies)


@pytest.mark.parametrize("override,version", [("", "v2"), ("o-1", "")])
def test_edge_corpus(ctx, override, version):
    bodies = G.edge_corpus() + G.class_bound_bodies()
    tally = check(bodies, run_paths(ctx, bodies, override, version), override, version)
    report("edge corpus (override %r)" % override, tally)
    assert tally[(OK, 0)] and sum(n for (s, _), n in tally.items() if s == E400) and sum(n for (s, _), n in tally.items() if s == DECLINED)
    big = G.class_bound_bodies()[-1]
    assert len(big) > 65536 and ctx.chat_translate(ctx.cfg(SCHEMA, api_version="v2"), [big])[0]["reason"] == R_TOO_LARGE


def test_mutants(ctx):
    seeds = [c["body"].encode() for c in G.GOLD["parse_body"][1:]] + [b for b in G.realistic_corpus(200, seed=3) if len(b) < 900][:30]
    bodies = [m for s in seeds for m in E.mutants(s)]
    tally = check(bodies, run_paths(ctx, bodies, batcher=False))
    report("mutants (%d from %d bodies)" % (len(bodies), len(seeds)), tally)


def test_document_capacity(ctx):
    """per size class, the most one-character documents the index stage holds is OK and one more declines with AIGW_R_TOKENS;
    the same for the fused kernel (its own capacity) on bodies up to 5120 bytes"""
    cfg = ctx.cfg(SCHEMA, api_version="v2")
    found = {}
    for label, small, ktok, classes in (("pipeline", 0, E.KTOK, E.CLASSES), ("fused", 1 << 20, {2048: E.SMALL_KTOK, 5120: E.SMALL_KTOK}, (2048, 5120))):
        cases = G.capacity_cases(ktok, classes)
        try:
            ctx.chat_set_small_batch(small)
            res = ctx.chat_translate(cfg, [b for _, _, fit, over in cases for b in (fit, over)])
        finally:
            ctx.chat_set_small_batch(-1)
        for j, (c, k, fit, over) in enumerate(cases):
            g_fit, g_over = res[2 * j], res[2 * j + 1]
            assert (g_fit["status"], g_fit["reason"], g_fit["path"]) == (OK, 0, b"/v2/rerank"), (label, c, k, g_fit)
            assert (g_over["status"], g_over["reason"]) == (DECLINED, R_TOKENS), (label, c, k + 1, g_over)
            found[(label, c)] = (k, len(fit))
    print("\nmost one-character documents per size class (documents, body bytes):", found)


def test_long_version_declines(ctx):
    """a version whose cleaned path does not fit the 128-byte path buffer declines; 120 characters still fit"""
    body = b'{"model":"m"}'
    ok = ctx.chat_translate(ctx.cfg(SCHEMA, api_version="v" * 120), [body])[0]
    assert (ok["status"], ok["path"]) == (OK, b"/" + b"v" * 120 + b"/rerank")
    assert ctx.chat_translate(ctx.cfg(SCHEMA, api_version="v" * 121), [body])[0]["status"] == DECLINED


# ================================================================ buffered responses
def _unpack(r):
    m = int(r["mask"])
    assert not m & ~7
    return (int(r["input"]) if m & 1 else -1, int(r["output"]) if m & 2 else -1, int(r["total"]) if m & 4 else -1)


def _check_usage(res, bodies, costs=None):
    tally = collections.Counter()
    for i, b in enumerate(bodies):
        v, u = Q.response_usage(b)
        r = res[i]
        st = int(r["status"])
        tally[st] += 1
        assert int(r["model_len"]) == 0, i
        if st == DECLINED:
            assert v != Q.OK, (i, b[:300])
        elif st == INTERNAL:
            assert v == Q.FAIL, (i, b[:300])
        else:
            assert st == OK and v == Q.OK and _unpack(r) == u, (i, b[:300], _unpack(r), u, v)
            if costs is not None:   # input, cached, cache_creation, output, total, reasoning
                assert [int(x) for x in costs[i]] == [max(u[0], 0), 0, 0, max(u[1], 0), max(u[2], 0), 0], i
        if v == Q.OK:
            assert st == OK, (i, b[:300], st)   # nothing the oracle decodes is declined: the float conversion is exact
    return tally


def test_response_goldens(ctx):
    import aigw_b200 as A
    bodies = [c["body"].encode() for c in G.GOLD["response_body"]]
    res, _ = ctx.response_usage_host(*A.pack_bodies(bodies), rerank=True)
    for c, r in zip(G.GOLD["response_body"], res):
        if c["error"]:
            assert int(r["status"]) == INTERNAL, c["name"]
        else:
            assert int(r["status"]) == OK and _unpack(r) == (c["input"], c["output"], c["total"]), c["name"]


def test_response_corpus_host(ctx):
    import aigw_b200 as A
    bodies = G.response_corpus()
    res, costs = ctx.response_usage_host(*A.pack_bodies(bodies), cost_types=(0, 1, 2, 3, 4, 5), rerank=True)
    tally = _check_usage(res, bodies, costs)
    print("\nrerank buffered (host): %d bodies, by status %s" % (len(bodies), dict(tally)))
    assert tally[OK] > 1900 and tally[INTERNAL] > 50 and tally[DECLINED] > 20
    wrap = bodies.index(G.token_response(b"4294967295", b"1"))
    assert _unpack(res[wrap]) == (4294967295, 1, 0)


def test_response_corpus_device(ctx):
    import ctypes as C
    import aigw_b200 as A
    from aigw_b200 import capi
    bodies = G.response_corpus()
    arena, offs, lens = A.pack_bodies(bodies)
    n = len(bodies)
    L, h = ctx.L, ctx.h
    d_b, d_o, d_l, d_r = (L.aigw_device_alloc(h, max(16, x)) for x in (arena.nbytes, offs.nbytes, lens.nbytes, n * capi.SseResult.itemsize))
    try:
        for d, a in ((d_b, arena), (d_o, offs), (d_l, lens)):
            assert L.aigw_memcpy_h2d(h, d, a.ctypes.data, a.nbytes) == 0
        ms = C.c_float(0)
        assert L.aigw_rerank_response_usage_device(h, d_b, d_o, d_l, n, d_r, None, C.byref(ms)) == 0
        assert L.aigw_sync(h) == 0
        res = np.zeros(n, dtype=capi.SseResult)
        assert L.aigw_memcpy_d2h(h, res.ctypes.data, d_r, res.nbytes) == 0
    finally:
        for d in (d_b, d_o, d_l, d_r):
            L.aigw_device_free(h, d)
    _check_usage(res, bodies)


# ================================================================ error bodies
@pytest.mark.parametrize("force", [True, False])
def test_error_bodies(ctx, force):
    bodies = G.error_bodies()
    for small in (0, 1 << 20):
        try:
            ctx.chat_set_small_batch(small)
            res = ctx.chat_translate(ctx.cfg("resp-error-cohere", model_override="503", force=force), bodies)
        finally:
            ctx.chat_set_small_batch(-1)
        for b, g in zip(bodies, res):
            v, out = Q.response_error(b, force)
            if v == Q.OK and out is not None:
                assert (g["status"], g["body"]) == (OK, out), (small, b[:100], g)
            else:
                assert g["status"] == DECLINED, (small, b[:100], g)   # forwarded untouched, non-ASCII, or the empty body
        assert res[bodies.index(b"")]["status"] == DECLINED


@pytest.mark.parametrize("override,force", [("rerank-english-v3", False), ("", True)])
def test_path_straddles(ctx, override, force):
    """versions of 1-20 characters put the end of ":path" (and so the first body op) at every offset of a 16-byte output chunk; the
    fused kernel and the pipeline give the oracle's bytes at each (the fused kernel's emit loop is the one ptxas -O3 miscompiles)"""
    body = b'{"model":"m","query":"q","documents":["a","b"],"top_n":1}'
    for n in range(1, 21):
        version = "v" * n
        v, path, out, _ = Q.translate(body, override, version, force)
        cfg = ctx.cfg(SCHEMA, model_override=override or None, force=force, api_version=version)
        for small in (0, 1 << 20):
            try:
                ctx.chat_set_small_batch(small)
                g = ctx.chat_translate(cfg, [body])[0]
            finally:
                ctx.chat_set_small_batch(-1)
            assert (g["status"], g["path"].decode(), g["body"]) == (OK, path, out), (version, small, g)
