"""/v1/responses requests of any size through aigw_responses_translate_large_{host,device}: the translate pass's answers on its own
corpora (test_responses_request_gpu.py), the oracle's bytes on long agent sessions (test_responses_large_cpu.py), 400s deep in
large bodies, the limits, malformed bytes on the scan's boundaries, other schemas, the device form's output space and call
composition."""
import numpy as np
import pytest

import _responses_request_oracle as Q
import test_responses_large_cpu as L
import test_responses_request_cpu as G
import test_responses_request_gpu as RG
import test_translate_edges_cpu as E

pytestmark = pytest.mark.gpu

OK, E400, DECLINED = 0, 1, 4
SCHEMA = "responses-openai"
R_TOO_LARGE, R_CTRL, R_ESCAPE, R_TOKENS, R_OUT_SPACE, R_DEPTH, R_SCHEMA = 1, 3, 4, 5, 8, 16, 19
CAPACITY = (R_TOO_LARGE, R_TOKENS, 6, 7, R_OUT_SPACE, 18)   # the translate pass's own capacity declines
EXTRA = (R_ESCAPE, R_TOO_LARGE, R_TOKENS, R_DEPTH)          # the declines the header lists beyond the translate pass's
KEYS = ("status", "path", "body", "body_kind", "model", "stream", "flags")


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def cfg(ctx, override="", prefix="v1", force=False, schema=SCHEMA):
    return ctx.cfg(schema, model_override=override or None, force=force, prefix=prefix)


def run(ctx, fn, c, bodies):
    import aigw_b200 as A
    arena, offs, lens = A.pack_bodies(bodies)
    res, out, _ = fn(c, arena, offs, lens)
    recs = ctx._records(bodies, res, out)
    for r, x in zip(recs, res):
        r["flags"] = int(x["flags"])
    return recs


def large(ctx, c, bodies):
    return run(ctx, ctx.responses_translate_large_host, c, bodies)


def small(ctx, c, bodies):
    ctx.chat_set_small_batch(0)
    try:
        return run(ctx, ctx.chat_translate_host, c, bodies)
    finally:
        ctx.chat_set_small_batch(-1)


def same_as_translate_pass(bodies, got, ref, label):
    """equal to group 10, or declined with a listed reason; returns (compared, extra declines)"""
    compared = extra = 0
    for b, g, h in zip(bodies, got, ref):
        if h["status"] == DECLINED and h["reason"] in CAPACITY:
            continue
        if g["status"] == DECLINED and h["status"] != DECLINED:
            assert g["reason"] in EXTRA, (label, b[:300], g["reason"], h["status"])
            extra += 1
            continue
        assert all(g[k] == h[k] for k in KEYS), (label, b[:300], {k: (g[k], h[k]) for k in KEYS if g[k] != h[k]}, g["reason"], h["reason"])
        compared += 1
    return compared, extra


def _translate_corpora():
    unions = [u["wrapped"].encode() for u in G.GOLD["unions"]]
    goldens = unions + [c["body"].encode() for c in G.GOLD["parse_body"]] + [c["body"].encode() for c in G.GOLD["request_body"]]
    goldens += [G.UPSTREAM[n]["requestBody"].encode() for n in ("openai - /v1/responses", "openai - /v1/responses - stream")]
    mutants = []
    for k, s in enumerate(G.mutation_seeds()):
        ms = list(E.mutants(s))
        mutants += ms if len(s) < 400 else ms[k % 7::7]
    return {"goldens": goldens, "realistic": G.realistic_corpus(2000), "edges": G.edge_corpus() + G.class_bound_bodies(), "mutants": mutants}


def test_translate_corpora(ctx):
    corpora = _translate_corpora()
    totals = {}
    for override, prefix, force in RG.CONFIGS:
        c = cfg(ctx, override, prefix, force)
        for name, bodies in corpora.items():
            n, extra = same_as_translate_pass(bodies, large(ctx, c, bodies), small(ctx, c, bodies), (override, prefix, force, name))
            t = totals.setdefault(name, [0, 0]); t[0] += n; t[1] += extra
    print("\ncompared with the translate pass (bodies, extra declines):", totals)
    assert totals["goldens"][1] == 0 and totals["realistic"][1] == 0
    assert totals["realistic"][0] == 2000 * len(RG.CONFIGS)


def check_oracle(bodies, got, override="", prefix="v1", force=False):
    for b, g in zip(bodies, got):
        v, path, out, model, stream = L.expect(b, override, prefix, force)
        assert g["status"] == OK and v == Q.OK, (len(b), g["status"], g["reason"], v)
        assert g["path"].decode() == path and g["body_kind"] == (0 if out is None else 1), (len(b), g["path"], path)
        assert g["model"] == model and g["stream"] == stream and g["flags"] == int(stream), (len(b), g["model"][:40], model[:40])
        assert g["body"] == (out or b""), (len(b), len(g["body"]), len(out or b""))


@pytest.mark.parametrize("override,prefix,force", [("", "v1", False), ("gpt-5-mini", "v1", False), ("", "v1", True), ("", "custom/api/", False)])
def test_large_realistic(ctx, override, prefix, force):
    bodies = list(L.realistic_corpus())
    check_oracle(bodies, large(ctx, cfg(ctx, override, prefix, force), bodies), override, prefix, force)


def test_large_errors_are_400(ctx):
    import json
    base = L.long_session(3, 1200 << 10)
    assert base.endswith(b"]}")   # input is the last member
    j = json.loads(base)
    j["input"].append({"type": "function_call", "call_id": 5, "name": "f", "arguments": "{}"})
    bad = [json.dumps(j, separators=(",", ":")).encode(),                             # a type error in the last input item
           base[:-1] + b',"max_output_tokens":"many"}',                              # a wrong-typed top-level member after 1 MB of items
           base[:-3], base[:len(base) // 2],                                          # truncations
           base + b"x", base + b" {}"]                                                # trailing bytes
    for b in bad:
        assert L.verdict(b)[0] == Q.FAIL, b[-80:]
    got = large(ctx, cfg(ctx), bad)
    assert [g["status"] for g in got] == [E400] * len(bad), [(g["status"], g["reason"]) for g in got]


def test_boundaries(ctx):
    bodies = list(L.boundary_bodies())
    for override, prefix, force in [("ovr", "v1", False), ("", "v1", True), ("", "custom/api/", False)]:
        c = cfg(ctx, override, prefix, force)
        got = large(ctx, c, bodies)
        for b, g in zip(bodies, got):
            v = L.verdict(b)[0]
            if v == Q.OK:
                check_oracle([b], [g], override, prefix, force)
            else:
                assert g["status"] == E400 and v == Q.FAIL, (b[:80], g["status"], g["reason"])
        short = [b for b in bodies if len(b) <= 65536]
        n, extra = same_as_translate_pass(short, large(ctx, c, short), small(ctx, c, short), "boundaries")
        assert extra == 0 and n == len(short)


def test_limits(ctx):
    c = cfg(ctx, "o")
    g = large(ctx, c, [L.deep(48), L.deep(49)])
    assert (g[0]["status"], g[1]["status"], g[1]["reason"]) == (OK, DECLINED, R_DEPTH)
    check_oracle([L.deep(48)], g[:1], "o")
    assert small(ctx, c, [L.deep(49)])[0]["reason"] == R_DEPTH
    big = L.near_16mib()
    g = large(ctx, c, [big, big + b" "])
    check_oracle([big], g[:1], "o")
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_TOO_LARGE)
    at, over = L.token_edge(L.TOKEN_K, L.TOKEN_LEN), L.token_edge(L.TOKEN_K + 1, L.TOKEN_LEN)
    g = large(ctx, c, [at, over])
    check_oracle([at], g[:1], "o")
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_TOKENS)


def test_scan_defects(ctx):
    """malformed bytes on the thread, warp and tile boundaries of four probes, and backslash runs across them: a GPU OK is the
    oracle's record, a GPU 400 the oracle's failure, and a decline of a body the oracle accepts has a listed reason"""
    items = [(label, b) for label, _, b in L.probe_corpus()] + list(L.run_corpus())
    bodies = [b for _, b in items]
    got = large(ctx, cfg(ctx, "ovr"), bodies)
    tally = {}
    for (label, b), g in zip(items, got):
        v = L.verdict(b)[0]
        if g["status"] == OK:
            check_oracle([b], [g], "ovr")
        elif g["status"] == E400:
            assert v == Q.FAIL, (label, g["reason"])
        else:
            assert g["status"] == DECLINED and (v != Q.OK or g["reason"] in EXTRA), (label, g["reason"], v)
        if label.startswith("run"):
            assert (g["status"] == OK) == label.endswith(" valid"), (label, g["status"], g["reason"])
        tally[(g["status"], g["reason"])] = tally.get((g["status"], g["reason"]), 0) + 1
    print("\nscan defects (%d bodies): %s" % (len(bodies), sorted(tally.items())))
    assert tally.get((OK, 0), 0) > 100 and sum(n for (s, _), n in tally.items() if s == E400) > 500


def test_other_schemas_decline(ctx):
    bodies = [L.long_session(5, 100 << 10), b'{"model":"m","input":"hi"}']
    for schema in ["openai", "completions-openai", "rerank-cohere"] + [128 | base for base in (1, 2, 3, 4, 5, 6)]:
        got = large(ctx, ctx.cfg(schema), bodies)
        assert all((g["status"], g["reason"]) == (DECLINED, R_SCHEMA) for g in got), schema


def test_device_out_space(ctx):
    import torch
    import aigw_b200 as A
    bodies = [L.long_session(11, 300 << 10), L.long_session(12, 90 << 10)]
    arena, offs, lens = A.pack_bodies(bodies)
    c = cfg(ctx, "ovr")
    d_b = torch.from_numpy(arena).cuda(); d_o = torch.from_numpy(offs.astype(np.uint64).view(np.int64)).cuda(); d_l = torch.from_numpy(lens.astype(np.uint32).view(np.int32)).cuda()
    host = large(ctx, c, bodies)
    for cap in (16, len(bodies[1]) + 4096):
        d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        d_r = torch.zeros(len(bodies) * 32, dtype=torch.uint8, device="cuda"); d_u = torch.zeros(1, dtype=torch.int64, device="cuda")
        ctx.responses_translate_large_device(c, d_b.data_ptr(), d_o.data_ptr(), d_l.data_ptr(), len(bodies), int(lens.max()), d_out.data_ptr(), cap, d_r.data_ptr(), d_u.data_ptr())
        res = d_r.cpu().numpy().view(A.DocResult)
        for i, x in enumerate(res):
            if int(x["status"]) == OK:
                assert int(x["body_len"]) == len(host[i]["body"])
            else:
                assert (int(x["status"]), int(x["reason"])) == (DECLINED, R_OUT_SPACE)
                assert int(x["body_len"]) == len(host[i]["path"]) + len(host[i]["body"])
        if cap == 16:
            assert all(int(x["status"]) == DECLINED for x in res)


def test_mixed_call(ctx):
    rng = np.random.default_rng(5)
    mixed = [L.long_session(40 + i, int(rng.integers(1 << 10, 3 << 20)), L.STREAM_FORMS[i % 4]) for i in range(10)]
    mixed += G.realistic_corpus(50, seed=9) + G.edge_corpus()[:80]
    c = cfg(ctx, "ovr")
    whole = large(ctx, c, mixed)
    order = list(rng.permutation(len(mixed)))
    rev = large(ctx, c, [mixed[i] for i in order])
    cut = len(mixed) // 3
    split = large(ctx, c, mixed[:cut]) + large(ctx, c, mixed[cut:])
    for i, j in enumerate(order):
        assert all(rev[i][k] == whole[j][k] for k in KEYS)
    for a, b in zip(whole, split):
        assert all(a[k] == b[k] for k in KEYS)
    assert sum(g["status"] == OK for g in whole[:10]) == 10
