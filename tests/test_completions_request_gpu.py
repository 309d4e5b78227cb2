"""/v1/completions requests (AIGW_SCHEMA_COMPLETIONS | OpenAI) through every entry point of the translate pass: the host call, the
fused small-batch kernel, the device call, the device-mapped call and the batcher.  Every path is checked against the oracle
(tests/_completions_request_oracle.py):
  * a GPU OK is an oracle OK with the same ":path", body bytes, body kind, model span and stream flag;
  * a GPU 400 is an oracle failure;
  * a GPU decline is an input the oracle fails or puts outside the subset, or a capacity / size decline.
The paths agree with each other wherever none of them declined for capacity: the fused kernel's token capacity (640) differs
from the pipeline's in the 2048-byte class (512).  Corpora: tests/test_completions_request_cpu.py."""
import collections

import pytest

import _completions_request_oracle as Q
from _responses_request_oracle import _raw_limits
import test_completions_request_cpu as G
import test_responses_request_gpu as RG
import test_translate_edges_cpu as E
import test_translate_edges_gpu as EG

pytestmark = pytest.mark.gpu

OK, E400, DECLINED = 0, 1, 4
SCHEMA = "completions-openai"
R_TOO_LARGE, R_TOKENS, R_SCHEMA = 1, 5, 19
CAPACITY = (R_TOKENS, 6, 7)   # tokens, ops, scratch
CONFIGS = [("", "v1", False), ("gpt-4-turbo", "v1", False), ("", "v1", True), ("o-1", "custom/api/", False)]


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.chat_set_small_batch(-1)
    c.close()


def run_paths(ctx, bodies, override="", prefix="v1", force=False, batcher=True):
    cfg = ctx.cfg(SCHEMA, model_override=override or None, force=force, prefix=prefix)
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


def check(bodies, paths, override="", prefix="v1", force=False):
    """the three rules on every path, the paths equal where none declined for capacity; → Counter of (status, reason) of the host call"""
    tally = collections.Counter()
    for i, body in enumerate(bodies):
        v, path, out, model, stream = Q.translate(body, override, prefix, force)
        got = {name: r[i] for name, r in paths.items() if r[i] is not None}
        tally[(got["host"]["status"], got["host"]["reason"])] += 1
        for name, g in got.items():
            where = (name, body[:300], g["status"], g["reason"], v)
            if g["status"] == OK:
                assert v == Q.OK, where
                assert g["path"].decode() == path and g["body"] == (out or b"") and g["body_kind"] == (0 if out is None else 1), (where, g, out)
                if "model" in g:
                    assert g["model"] == model and g["stream"] == stream, (where, g, model, stream)
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


@pytest.mark.parametrize("override,prefix,force", CONFIGS)
def test_goldens(ctx, override, prefix, force):
    unions = [u["wrapped"].encode() for u in G.GOLD["unions"]]
    cassettes = [c["body"].encode() for c in G.GOLD["cassettes"]]
    bodies = unions + [c["body"].encode() for c in G.GOLD["parse_body"]] + [c["body"].encode() for c in G.GOLD["request_body"]] + cassettes
    paths = run_paths(ctx, bodies, override, prefix, force)
    report("goldens %r" % ((override, prefix, force),), check(bodies, paths, override, prefix, force))
    for i, b in enumerate(bodies):   # what the oracle decodes is OK, byte-exact (checked above); null prompts decline, errors are 400
        v = Q.parse_body(b)[0]
        want = {Q.OK: OK, Q.FAIL: E400, Q.OUT: DECLINED}[v]
        assert all(r[i] is None or r[i]["status"] == want for r in paths.values()), (b, [r[i] for r in paths.values()])
    for b in cassettes:
        assert paths["host"][bodies.index(b)]["status"] == OK
    for c in G.GOLD["request_body"]:
        if c["override"] == override and c["force"] == force and prefix == "v1":
            g = paths["host"][bodies.index(c["body"].encode())]
            assert g["path"] == b"/v1/completions" and g["stream"] == c.get("stream", False)


def test_other_backends_decline(ctx):
    body = b'{"model":"m","prompt":"hi"}'
    for schema in (257, 258, 259, 260, 261, 262, 256 | 128, 256 | 64, 256 | 32):
        for r in ctx.chat_translate(ctx.cfg(schema), [body]):
            assert (r["status"], r["reason"]) == (DECLINED, R_SCHEMA), (schema, r)


@pytest.mark.parametrize("override", ["", "gpt-5-mini"])
def test_realistic_corpus(ctx, override):
    """every body decodes; the only declines are token-id prompts beyond the index stage's token capacity"""
    bodies = G.realistic_corpus(2000)
    paths = run_paths(ctx, bodies, override)
    tally = check(bodies, paths, override)
    report("realistic corpus (override %r)" % override, tally)
    assert set(tally) <= {(OK, 0), (DECLINED, R_TOKENS)}, tally
    for i, b in enumerate(bodies):
        over = E.count_tokens(b) > E.KTOK[E.class_of(len(b))]
        assert (paths["host"][i]["status"] == DECLINED) == over, (len(b), E.count_tokens(b))
    assert tally[(OK, 0)] >= 0.98 * len(bodies)


@pytest.mark.parametrize("override", ["", "o-1"])
def test_edge_corpus(ctx, override):
    bodies = G.edge_corpus() + G.class_bound_bodies()
    tally = check(bodies, run_paths(ctx, bodies, override), override)
    report("edge corpus (override %r)" % override, tally)
    assert tally[(OK, 0)] and sum(n for (s, _), n in tally.items() if s == E400) and sum(n for (s, _), n in tally.items() if s == DECLINED)


def indexable(body):
    """no raw control character in a string and no nesting beyond what the index stage takes: its declines come first"""
    ctrl, depth = _raw_limits(body)
    return not ctrl and depth <= Q.MAX_DEPTH


def test_edge_verdicts(ctx):
    """the edge corpus inside the restated subset gets exactly the oracle's verdict: OK, or 400 for a decode failure"""
    bodies = [b for b in G.edge_corpus() if Q.parse_body(b)[0] != Q.OUT and indexable(b)]
    res = ctx.chat_translate(ctx.cfg(SCHEMA), bodies)
    for b, g in zip(bodies, res):
        want = OK if Q.parse_body(b)[0] == Q.OK else E400
        assert g["status"] == want, (b[:200], g["status"], g["reason"])


def test_mutants(ctx):
    seeds = G.mutation_seeds()
    bodies = []
    for k, s in enumerate(seeds):
        ms = list(E.mutants(s))
        bodies += ms if len(s) < 400 else ms[k % 5::5]
    tally = check(bodies, run_paths(ctx, bodies, batcher=False))
    report("mutants (%d from %d bodies)" % (len(bodies), len(seeds)), tally)


def test_token_capacity(ctx):
    """per size class, the longest compact token-id prompt the index stage holds is OK and one more id declines with
    AIGW_R_TOKENS; the same for the fused kernel (its own capacity) on bodies up to 5120 bytes"""
    cfg = ctx.cfg(SCHEMA)
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
            assert (g_fit["status"], g_fit["reason"], g_fit["body_kind"]) == (OK, 0, 0), (label, c, k, g_fit)
            assert g_fit["path"] == b"/v1/completions" and g_fit["model"] == b"m"
            assert (g_over["status"], g_over["reason"]) == (DECLINED, R_TOKENS), (label, c, k + 1, g_over)
            found[(label, c)] = (k, len(fit))
        if label == "pipeline":
            for c in E.CLASSES:   # the device call, one class per call
                _, k, fit, over = cases[E.CLASSES.index(c)]
                g = EG.device_translate(ctx, cfg, [fit, over], c)
                assert (g[0]["status"], g[1]["status"], g[1]["reason"]) == (OK, DECLINED, R_TOKENS), (c, g)
    print("\nlongest compact five-digit token-id prompt per size class (ids, body bytes):", found)


@pytest.mark.parametrize("override,force", [("gpt-4-turbo", False), ("", True)])
def test_path_straddles(ctx, override, force):
    """prefixes of 1-20 characters put the end of ":path" (and so the first body op) at every offset of a 16-byte output chunk;
    the fused kernel and the pipeline give the oracle's bytes at each, for /v1/completions and, as a control, /v1/responses"""
    import _responses_request_oracle as RQ
    for schema, oracle, body in (("completions-openai", Q, b'{"model":"m","prompt":"p","max_tokens":7}'), ("responses-openai", RQ, b'{"model":"m","input":"p"}')):
        for n in range(1, 21):
            prefix = "v" * n
            v, path, out, _, _ = oracle.translate(body, override, prefix, force)
            cfg = ctx.cfg(schema, model_override=override or None, force=force, prefix=prefix)
            for small in (0, 1 << 20):
                try:
                    ctx.chat_set_small_batch(small)
                    g = ctx.chat_translate(cfg, [body])[0]
                finally:
                    ctx.chat_set_small_batch(-1)
                assert (g["status"], g["path"].decode(), g["body"]) == (OK, path, out), (schema, prefix, small, g)
