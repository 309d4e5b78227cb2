"""/v1/completions requests of any size through aigw_completions_translate_large_{host,device}: the translate pass's answers on its
own corpora (test_completions_request_gpu.py), the token-id prompts it declines for capacity, the oracle's bytes on large requests
(test_completions_large_cpu.py), 400s deep in large bodies, the boundaries, the limits, probes that break a flat prompt on them,
flags that must not outlive their request in a reused slice, other schemas, the device form's output space and call composition."""
import numpy as np
import pytest

import _completions_request_oracle as Q
import test_completions_large_cpu as L
import test_completions_request_cpu as G
import test_completions_request_gpu as CG
import test_translate_edges_cpu as E

pytestmark = pytest.mark.gpu

OK, E400, DECLINED = 0, 1, 4
SCHEMA = "completions-openai"
R_TOO_LARGE, R_ESCAPE, R_TOKENS, R_OUT_SPACE, R_DEPTH, R_SCHEMA = 1, 4, 5, 8, 16, 19
CAPACITY = (R_TOO_LARGE, R_TOKENS, 6, 7, R_OUT_SPACE, 18)   # the translate pass's own capacity declines
EXTRA = (R_ESCAPE, R_TOO_LARGE, R_TOKENS, R_DEPTH)          # the declines the header lists beyond the translate pass's
KEYS = ("status", "path", "body", "body_kind", "model", "stream", "flags")
WANT = {Q.OK: OK, Q.FAIL: E400, Q.OUT: DECLINED}


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
    return run(ctx, ctx.completions_translate_large_host, c, bodies)


def small(ctx, c, bodies):
    ctx.chat_set_small_batch(0)
    try:
        return run(ctx, ctx.chat_translate_host, c, bodies)
    finally:
        ctx.chat_set_small_batch(-1)


def check_oracle(bodies, got, override="", prefix="v1", force=False):
    for b, g in zip(bodies, got):
        v, path, out, model, stream = L.expect(b, override, prefix, force)
        assert g["status"] == OK and v == Q.OK, (len(b), b[:200], g["status"], g["reason"], v)
        assert g["path"].decode() == path and g["body_kind"] == (0 if out is None else 1), (len(b), g["path"], path)
        assert g["model"] == model and g["stream"] == stream and g["flags"] == int(stream), (len(b), g["model"][:40], model[:40])
        assert g["body"] == (out or b""), (len(b), len(g["body"]), len(out or b""))


def same_as_translate_pass(bodies, got, ref, label, cfg_args):
    """equal to group 11, or declined with a listed reason; a body the translate pass declines with AIGW_R_TOKENS and the oracle
    accepts must be the oracle's record.  → (compared, extra declines, token-capacity bodies answered)"""
    compared = extra = answered = 0
    for b, g, h in zip(bodies, got, ref):
        if h["status"] == DECLINED and h["reason"] == R_TOKENS and L.verdict(b)[0] == Q.OK:
            check_oracle([b], [g], *cfg_args)
            answered += 1
            continue
        if h["status"] == DECLINED and h["reason"] in CAPACITY:
            continue
        if g["status"] == DECLINED and h["status"] != DECLINED:
            assert g["reason"] in EXTRA, (label, b[:300], g["reason"], h["status"])
            extra += 1
            continue
        assert all(g[k] == h[k] for k in KEYS), (label, b[:300], {k: (g[k], h[k]) for k in KEYS if g[k] != h[k]}, g["reason"], h["reason"])
        compared += 1
    return compared, extra, answered


def _translate_corpora():
    unions = [u["wrapped"].encode() for u in G.GOLD["unions"]]
    goldens = unions + [c["body"].encode() for c in G.GOLD["parse_body"]] + [c["body"].encode() for c in G.GOLD["request_body"]]
    goldens += [c["body"].encode() for c in G.GOLD["cassettes"]]
    mutants = []
    for k, s in enumerate(G.mutation_seeds()):
        ms = list(E.mutants(s))
        mutants += ms if len(s) < 400 else ms[k % 5::5]
    return {"goldens": goldens, "realistic": G.realistic_corpus(2000), "edges": G.edge_corpus() + G.class_bound_bodies(), "mutants": mutants}


def test_translate_corpora(ctx):
    corpora = _translate_corpora()
    totals = {}
    for override, prefix, force in CG.CONFIGS:
        c = cfg(ctx, override, prefix, force)
        for name, bodies in corpora.items():
            got = same_as_translate_pass(bodies, large(ctx, c, bodies), small(ctx, c, bodies), (override, prefix, force, name), (override, prefix, force))
            t = totals.setdefault(name, [0, 0, 0])
            for i in range(3):
                t[i] += got[i]
    print("\ncompared with the translate pass (bodies, extra declines, token-capacity declines answered):", totals)
    assert totals["goldens"][1] == 0 and totals["realistic"][1] == 0
    # every realistic body is compared, or is a token-id prompt the translate pass declines and this call answers exactly
    assert totals["realistic"][0] + totals["realistic"][2] == 2000 * len(CG.CONFIGS) and totals["realistic"][2] > 0


def test_token_capacity(ctx):
    """the bodies one id beyond the translate pass's token capacity in every size class are OK here, and so are those at it"""
    c = cfg(ctx)
    cases = G.capacity_cases()
    bodies = [b for _, _, fit, over in cases for b in (fit, over)]
    ref = small(ctx, c, bodies)
    assert [(r["status"], r["reason"]) for r in ref[1::2]] == [(DECLINED, R_TOKENS)] * len(cases)
    check_oracle(bodies, large(ctx, c, bodies))


@pytest.mark.parametrize("override,prefix,force", [("", "v1", False), ("gpt-4-turbo", "v1", False), ("", "v1", True), ("", "custom/api/", False)])
def test_large_realistic(ctx, override, prefix, force):
    bodies = list(L.realistic_corpus())
    check_oracle(bodies, large(ctx, cfg(ctx, override, prefix, force), bodies), override, prefix, force)


def test_large_errors_are_400(ctx):
    ids = L._ids_text(150_000)   # a 1 MB flat prompt
    flat = b",".join(ids)
    base = b'{"model":"m","prompt":[' + flat + b'],"max_tokens":16}'
    batch = b'{"model":"m","prompt":[[' + flat[:len(flat) // 2].rstrip(b"0123456789").rstrip(b",") + b"],[" + flat[len(flat) // 2:].lstrip(b"0123456789").lstrip(b",")
    near_end = len(b'{"model":"m","prompt":[') + len(flat) - 20   # the third id from the end
    bad = [base[:near_end] + b"1.5" + base[near_end + 6:],                       # a fraction near the end of the flat prompt
           base[:near_end] + b"9223372036854775808" + base[near_end + 6:],       # an id beyond int64
           base[:near_end] + b"true" + base[near_end + 6:],                      # a bool among the ids
           base[:near_end] + b'"100000"' + base[near_end + 6:],                  # a string among the ids
           base[:-1] + b',"echo":"yes"}',                                        # a wrong-typed member after the prompt
           base[:-1] + b',"logit_bias":{"1":1.5}}',
           batch + b',2.5]],"max_tokens":16}',                                   # a fraction at the end of a batch's last inner array
           base[:-3], base[:len(base) // 2],                                     # truncations
           base + b"x", base + b" {}"]                                           # trailing bytes
    assert L.verdict(base)[0] == Q.OK and L.verdict(batch + b']]}')[0] == Q.OK
    for b in bad:
        assert L.verdict(b)[0] == Q.FAIL, b[-80:]
    got = large(ctx, cfg(ctx), bad + [base])
    assert [g["status"] for g in got] == [E400] * len(bad) + [OK], [(g["status"], g["reason"]) for g in got]


def test_boundaries(ctx):
    bodies = list(L.boundary_bodies())
    for override, prefix, force in [("ovr", "v1", False), ("", "v1", True), ("", "custom/api/", False)]:
        c = cfg(ctx, override, prefix, force)
        check_oracle(bodies, large(ctx, c, bodies), override, prefix, force)
        short = [b for b in bodies if len(b) <= 65536]
        n, extra, _ = same_as_translate_pass(short, large(ctx, c, short), small(ctx, c, short), "boundaries", (override, prefix, force))
        assert extra == 0 and n > len(short) // 2


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


@pytest.mark.parametrize("override", ["", "ovr"])
def test_probes(ctx, override):
    """every probe gets exactly the oracle's verdict: the record when it accepts, a 400 when it fails, a decline when the body
    is outside the subset (a float64 in stop with an exponent or more than 308 digits)"""
    items = list(L.probe_corpus())
    bodies = [b for _, b in items]
    got = large(ctx, cfg(ctx, override), bodies)
    for (label, b), g in zip(items, got):
        v = L.verdict(b)[0]
        assert g["status"] == WANT[v], (label, g["status"], g["reason"], v)
        if v == Q.OK:
            check_oracle([b], [g], override)


def test_no_stale_flags(ctx):
    """slices are reused request after request: a '[' that is flat and all-int64 in one request sits at the token index of a '['
    that is neither in the next.  An 8 MiB body in the call keeps the grid at about 15 CTAs, so each slice serves dozens of
    requests in an order the work counter decides."""
    ids = L._ids_text(400)
    flat = b'{"model":"m","prompt":[' + b",".join(ids) + b"]}"
    nested = b'{"model":"m","prompt":[' + b",".join(ids[:200]) + b",[1]," + b",".join(ids[201:]) + b"]}"
    wide = b'{"model":"m","prompt":[' + b",".join(ids[:200]) + b",1e2," + b",".join(ids[201:]) + b"]}"
    strs = b'{"model":"m","prompt":[' + b",".join(ids[:200]) + b',"s",' + b",".join(ids[201:]) + b"]}"
    kinds = [flat, nested, wide, strs]
    assert [WANT[L.verdict(b)[0]] for b in kinds] == [OK, E400, E400, E400]
    want = [(g["status"], g["reason"]) for g in large(ctx, cfg(ctx), kinds)]
    assert want[1:] == [(E400, 33)] * 3   # ParseBody's type error; a stale flag skips to a stale jump and reads a syntax error
    bodies = [L.realistic_corpus()[5]] + [kinds[i % 4] for i in range(2000)]
    assert len(bodies[0]) > 8_000_000
    got = large(ctx, cfg(ctx), bodies)
    assert got[0]["status"] == OK
    assert [(g["status"], g["reason"]) for g in got[1:]] == [want[i % 4] for i in range(2000)]
    check_oracle([flat], [got[1]])


def test_other_schemas_decline(ctx):
    bodies = [L.large_request(5, 100 << 10, "tokens"), b'{"model":"m","prompt":"hi"}']
    for schema in ["openai", "responses-openai", "rerank-cohere"] + [256 | base for base in (1, 2, 3, 4, 5, 6)]:
        got = large(ctx, ctx.cfg(schema), bodies)
        assert all((g["status"], g["reason"]) == (DECLINED, R_SCHEMA) for g in got), schema


def test_device_out_space(ctx):
    import torch
    import aigw_b200 as A
    bodies = [L.large_request(11, 300 << 10, "tokens"), L.large_request(12, 90 << 10, "fim")]
    arena, offs, lens = A.pack_bodies(bodies)
    c = cfg(ctx, "ovr")
    d_b = torch.from_numpy(arena).cuda(); d_o = torch.from_numpy(offs.astype(np.uint64).view(np.int64)).cuda(); d_l = torch.from_numpy(lens.astype(np.uint32).view(np.int32)).cuda()
    host = large(ctx, c, bodies)
    assert all(h["status"] == OK for h in host)
    for cap in (16, len(bodies[1]) + 4096):
        d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        d_r = torch.zeros(len(bodies) * 32, dtype=torch.uint8, device="cuda"); d_u = torch.zeros(1, dtype=torch.int64, device="cuda")
        ctx.completions_translate_large_device(c, d_b.data_ptr(), d_o.data_ptr(), d_l.data_ptr(), len(bodies), int(lens.max()), d_out.data_ptr(), cap, d_r.data_ptr(), d_u.data_ptr())
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
    mixed = [L.large_request(40 + i, int(rng.integers(1 << 10, 3 << 20)), L.KINDS[i % 4]) for i in range(10)]
    mixed += G.realistic_corpus(50, seed=9) + G.edge_corpus()[:80] + [b for _, b in L.probe_corpus()[:40]]
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
