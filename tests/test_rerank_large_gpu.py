"""Cohere /v2/rerank requests of any size through aigw_rerank_translate_large_{host,device}, against the oracle
(tests/_rerank_oracle.py) with the rules of test_rerank_gpu.check:
  * an OK is an oracle OK with the same ":path", body bytes, body kind and model span;
  * a 400 is an oracle failure;
  * a decline is an input the oracle fails or puts outside the subset, or a capacity decline.
And where the translate pass (aigw_chat_translate_host) did not decline for capacity or size, the large call gives its status,
":path", body, body kind and model span.  Corpora: test_rerank_cpu.py (the translate pass's) and test_rerank_large_cpu.py."""
import random

import numpy as np
import pytest

import _rerank_oracle as Q
import test_rerank_cpu as G
import test_rerank_gpu as RG
import test_rerank_large_cpu as L
import test_translate_edges_cpu as E

pytestmark = pytest.mark.gpu

OK, E400, DECLINED = 0, 1, 4
R_TOO_LARGE, R_TOKENS, R_OUT_SPACE, R_DEPTH = 1, 5, 8, 16
KEYS = ("status", "path", "body", "body_kind", "model")


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def cfg(ctx, override="", version="v2", force=False):
    return ctx.cfg(RG.SCHEMA, model_override=override or None, force=force, api_version=version or None)


def expect(body, override="", version="v2", force=False):
    """the oracle's (verdict, path, body or None, model), its verdict computed once per body"""
    from _oracle import body_mutate
    v, model = L.verdicts([body])[0]
    if v != Q.OK:
        return v, None, None, model
    out = None
    if override:
        rc, out = body_mutate(body, [], [("model", '"%s"' % override)])
        assert rc == 0
    elif force:
        out = body
    return v, Q.request_path(version), out, model


def check(bodies, got, override="", version="v2", force=False, capacity=(R_TOKENS,), labels=None):
    L.verdicts(bodies)   # all at once (in parallel) before the per-body loop
    tally = {}
    for i, (body, g) in enumerate(zip(bodies, got)):
        v, path, out, model = expect(body, override, version, force)
        where = (labels[i] if labels else i, body[:200], g["status"], g["reason"], v)
        if g["status"] == OK:
            assert v == Q.OK, where
            assert g["path"].decode() == path and g["body"] == (out or b"") and g["body_kind"] == (0 if out is None else 1), where
            assert g["model"] == model and g["stream"] is False, where
        elif g["status"] == E400:
            assert v == Q.FAIL, where
        else:
            assert g["status"] == DECLINED, where
            assert v != Q.OK or g["reason"] in capacity, where
        tally[(g["status"], g["reason"])] = tally.get((g["status"], g["reason"]), 0) + 1
    return tally


def device_translate(ctx, c, bodies, out_cap=None):
    """the device form on device buffers → the dicts of rerank_translate_large"""
    import aigw_b200 as A
    from aigw_b200 import capi
    arena, offs, lens = A.pack_bodies(bodies)
    n = len(bodies)
    need = sum((len(RG.Q.request_path("v2")) + 160 + len(b) + 16 + 15) // 16 * 16 for b in bodies)
    cap = need if out_cap is None else out_cap
    d_b, d_o, d_l, d_out, d_r, d_u = (ctx.dalloc(max(16, x)) for x in (arena.nbytes, offs.nbytes, lens.nbytes, cap, n * 32, 8))
    try:
        ctx.h2d(d_b, arena); ctx.h2d(d_o, offs); ctx.h2d(d_l, lens); ctx.memset(d_u, 0, 8)
        ctx.rerank_translate_large_device(c, d_b, d_o, d_l, n, int(lens.max()), d_out, cap, d_r, d_u)
        ctx.sync()
        res = np.zeros(n, dtype=capi.DocResult); used = np.zeros(1, dtype=np.uint64)
        ctx.d2h(res, d_r); ctx.d2h(used, d_u)
        out = np.zeros(max(16, min(int(used[0]), cap)), dtype=np.uint8)
        ctx.d2h(out, d_out, min(int(used[0]), cap))
    finally:
        for d in (d_b, d_o, d_l, d_out, d_r, d_u):
            ctx.dfree(d)
    return ctx._records(bodies, res, out)


# ================================================================ 1. the translate pass's corpora give the translate pass's answers
def _translate_corpora():
    seeds = [c["body"].encode() for c in G.GOLD["parse_body"][1:]] + [b for b in G.realistic_corpus(200, seed=3) if len(b) < 900][:30]
    return {
        "goldens": [c["body"].encode() for c in G.GOLD["parse_body"]] + [G.GOLD["request_body"][0]["body"].encode()],
        "realistic": G.realistic_corpus(2000),
        "edge": G.edge_corpus() + G.class_bound_bodies(),
        "mutants": [m for s in seeds for m in E.mutants(s)],
    }


@pytest.mark.parametrize("override,version,force", RG.CONFIGS)
def test_translate_corpora(ctx, override, version, force):
    c = cfg(ctx, override, version, force)
    for name, bodies in _translate_corpora().items():
        got = ctx.rerank_translate_large(c, bodies)
        ref = ctx.chat_translate(c, bodies)
        tally = check(bodies, got, override, version, force)
        same = 0
        for b, g, h in zip(bodies, got, ref):
            if h["status"] == DECLINED and (h["reason"] in RG.CAPACITY or h["reason"] == R_TOO_LARGE):
                continue
            assert all(g[k] == h[k] for k in KEYS), (name, b[:200], g, h)
            same += 1
        print("\n%s %r: %d bodies, %d compared with the translate pass, by (status, reason) %s" % (name, (override, version, force), len(bodies), same, tally))
        if name == "realistic":
            assert set(tally) == {(OK, 0)}, tally


# ================================================================ 2. large realistic requests: every one OK, byte-exact
@pytest.mark.parametrize("override,force", [("", False), ("rerank-v3.5", False), ("", True)])
def test_large_realistic(ctx, override, force):
    bodies = L.large_corpus()
    got = ctx.rerank_translate_large(cfg(ctx, override, force=force), bodies)
    assert check(bodies, got, override, force=force) == {(OK, 0): len(bodies)}


# ================================================================ 3. features at the scan's boundaries, and the splices
@pytest.mark.parametrize("override", ["", "rerank-v3.5"])
def test_boundaries(ctx, override):
    corpus = L.boundary_corpus()
    labels, bodies = [l for l, _ in corpus], [b for _, b in corpus]
    got = ctx.rerank_translate_large(cfg(ctx, override), bodies)
    tally = check(bodies, got, override, capacity=(), labels=labels)
    for l, b, g in zip(labels, bodies, got):
        name = l.split()[0]
        if name.startswith("run") or name in ("u_escape", "string_start", "string_end", "null_elem", "model"):
            assert g["status"] == OK, (l, g)    # no escaped quote ends a string, no valid escape is rejected
        elif name == "number_elem":
            assert g["status"] == E400, (l, g)
        else:
            assert g["status"] != OK, (l, g)
    print("\nboundary corpus: %d bodies, by (status, reason) %s" % (len(bodies), tally))


@pytest.mark.parametrize("override,force", [("", False), ("o-1", False), ("", True)])
def test_splices(ctx, override, force):
    bodies = L.splice_corpus()
    got = ctx.rerank_translate_large(cfg(ctx, override, force=force), bodies)
    check(bodies, got, override, force=force, capacity=())
    assert [g["status"] for g in got] == [OK] * 9 + [DECLINED, DECLINED, OK]
    if override:
        assert got[0]["body"].endswith(b'"model":"o-1"}') and got[2]["body"].startswith(b'{"query"') and got[4]["body"] == b'{"model":"o-1"}'


# ================================================================ 4. limits
def test_limits(ctx):
    c = cfg(ctx, "rerank-v3.5")
    near = L.near_limit_bodies()
    got = ctx.rerank_translate_large(c, [b for b, _ in near])
    for (b, accepted), g in zip(near, got):
        assert (g["status"], g["reason"]) == ((OK, 0) if accepted else (DECLINED, R_TOO_LARGE)), (len(b), g["status"], g["reason"])
    check([b for b, a in near if a], [g for (b, a), g in zip(near, got) if a], "rerank-v3.5")
    # token capacity: len / 4 + 1024 scan tokens
    n = 200000
    cap = n // 4 + 1024
    k = (cap - E.count_tokens(G.docs_body(1, n))) // 3 + 1
    while E.count_tokens(G.docs_body(k + 1, n)) <= cap:
        k += 1
    while E.count_tokens(G.docs_body(k, n)) > cap:
        k -= 1
    fit, over = G.docs_body(k, n), G.docs_body(k + 1, n)
    assert E.count_tokens(fit) <= cap < E.count_tokens(over)
    g_fit, g_over = ctx.rerank_translate_large(cfg(ctx), [fit]) + ctx.rerank_translate_large(cfg(ctx), [over])
    assert (g_fit["status"], g_fit["reason"]) == (OK, 0) and (g_over["status"], g_over["reason"]) == (DECLINED, R_TOKENS), (k, g_fit, g_over)
    # depth 48 is OK, 49 declines
    deep = [b'{"model":"m","x":' + b"[" * d + b"]" * d + b"}" for d in (47, 48)]
    assert [(g["status"], g["reason"]) for g in ctx.rerank_translate_large(cfg(ctx), deep)] == [(OK, 0), (DECLINED, R_DEPTH)]
    # an unknown member holding a 1 MiB nested value
    import json
    meta = json.dumps({"trace": [{"id": i, "tags": [None, True, "x" * 200, {"k": [1.5, -2, []]}]} for i in range(4500)]}).encode()
    assert len(meta) > 1 << 20
    big = b'{"model":"m","query":"q","metadata":' + meta + b',"documents":["a","b"],"top_n":1}'
    got = ctx.rerank_translate_large(cfg(ctx, "o"), [big])
    check([big], got, "o")
    assert (got[0]["status"], got[0]["reason"]) == (OK, 0), got[0]["reason"]


def test_out_space(ctx):
    """records that do not fit the device call's out_capacity decline with AIGW_R_OUT_SPACE; the others are intact"""
    bodies = L.large_corpus()[4:40]
    c = cfg(ctx, "rerank-v3.5")
    got = device_translate(ctx, c, bodies, out_cap=sum(len(b) for b in bodies) // 2)
    fit = [(b, g) for b, g in zip(bodies, got) if g["status"] == OK]
    assert fit and len(fit) < len(bodies)
    assert all((g["status"], g["reason"]) == (DECLINED, R_OUT_SPACE) for g in got if g["status"] != OK)
    check([b for b, _ in fit], [g for _, g in fit], "rerank-v3.5")


# ================================================================ 5. call composition, 6. the device form
def test_composition_and_device_form(ctx):
    r = random.Random(5)
    mixed = L.large_corpus()[4:60] + G.realistic_corpus(60, seed=8) + G.edge_corpus()[:40] + L.splice_corpus()[4:]
    r.shuffle(mixed)
    c = cfg(ctx, "rerank-v3.5")
    whole = ctx.rerank_translate_large(c, mixed)
    check(mixed, whole, "rerank-v3.5")
    order = list(range(len(mixed)))
    r.shuffle(order)
    rev = ctx.rerank_translate_large(c, [mixed[i] for i in order])
    cut = len(mixed) // 3
    split = ctx.rerank_translate_large(c, mixed[:cut]) + ctx.rerank_translate_large(c, mixed[cut:])
    dev = device_translate(ctx, c, mixed)
    for j, i in enumerate(order):
        assert all(rev[j][k] == whole[i][k] for k in KEYS + ("reason",)), i
    for i in range(len(mixed)):
        assert all(split[i][k] == whole[i][k] for k in KEYS + ("reason",)), i
        assert all(dev[i][k] == whole[i][k] for k in KEYS + ("reason",)), i


def test_other_schemas_decline(ctx):
    body = b'{"model":"m","query":"q","documents":["a"]}'
    for schema in (0, 512, 518, 519 | 256, 7, 32):
        g = ctx.rerank_translate_large(ctx.cfg(schema, api_version="v2"), [body, body * 2000])
        assert [(x["status"], x["reason"]) for x in g] == [(DECLINED, RG.R_SCHEMA)] * 2, schema
