"""/v1/embeddings requests of any size through aigw_embeddings_translate_large_{host,device}: the translate pass's answers on its
own corpora, the oracle's bytes on large requests (test_embeddings_large_cpu.py), the scan's boundaries, the limits, the device
form's output space and call composition."""
import json
import random

import numpy as np
import pytest

import _oracle as O
import test_embeddings_gpu as EG
import test_embeddings_large_cpu as L
import test_translate_edges_cpu as E

pytestmark = pytest.mark.gpu

OK, E400, DECLINED = 0, 1, 4
R_TOO_LARGE, R_ESCAPE, R_TOKENS, R_OPS, R_SCRATCH, R_OUT_SPACE, R_DEPTH, R_SCHEMA = 1, 4, 5, 6, 7, 8, 16, 19
CAPACITY = (R_TOKENS, R_OPS, R_SCRATCH)
KEYS = ("status", "reason", "path", "body", "body_kind", "model", "stream")
SCHEMAS = ["openai", "azure-openai", "gcp-vertexai", "aws-bedrock"]
VERSION = "2025-01-01-preview"


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def cfg(ctx, schema, override="", prefix=None, force=False):
    return ctx.cfg(EG.GPU_SCHEMA[schema], model_override=override or None, prefix=prefix if schema == "openai" else None,
                   api_version=VERSION if schema == "azure-openai" else None, force=force)


def escaped_key(body):
    """a key with a backslash at the root or inside an input item (the large call's documented decline)"""
    import re
    return re.search(rb'"(?:[^"\\]|\\.)*\\(?:[^"\\]|\\.)*"\s*:', body) is not None


def same_as_translate_pass(bodies, got, ref, label):
    compared, escaped = 0, 0
    for b, g, h in zip(bodies, got, ref):
        if h["status"] == DECLINED and (h["reason"] in CAPACITY or h["reason"] == R_TOO_LARGE):
            continue
        if g["status"] == DECLINED and g["reason"] == R_ESCAPE and h["reason"] != R_ESCAPE:
            assert escaped_key(b), (label, b[:200], g, h)
            escaped += 1
            continue
        assert all(g[k] == h[k] for k in KEYS if k != "reason"), (label, b[:300], g, h)
        if g["status"] != OK:
            assert g["reason"] == h["reason"], (label, b[:300], g, h)
        compared += 1
    return compared, escaped


def check_oracle(schema, bodies, got, override="", prefix="v1", force=False):
    for b, g in zip(bodies, got):
        t = O.embeddings_translate(schema, b, model_override=override, prefix=VERSION if schema == "azure-openai" else prefix, force=force)
        assert g["status"] == t.status == OK, (schema, b[:200], g["status"], g["reason"], t.status, t.err)
        assert g["path"].decode() == t.path and g["body_kind"] == t.body_kind and g["model"] == t.model, (b[:200], g["path"], t.path)
        if t.body_kind == 1:
            assert g["body"] == t.body, (schema, b[:200], len(g["body"]), len(t.body))


# ================================================================ 1. the translate pass's corpora give the translate pass's answers
def _translate_corpora():
    rng = np.random.default_rng(31)
    gold = [c["requestBody"].encode() for c in EG.EMB_CASES]
    seeds = gold + [EG.emb_body(rng) for _ in range(40)]
    return {"goldens": gold, "odd": EG.ODD, "emb_body": [EG.emb_body(np.random.default_rng(31)) for _ in range(1)] + [EG.emb_body(rng) for _ in range(3000)],
            "titan": [t[0] for t in EG.TITAN], "mutants": [m for s in seeds if len(s) < 2000 for m in E.mutants(s)]}


CONFIGS = [("", None, False), ("override-model", None, False), ("", None, True), ("", "v1", False), ("", "", False)]


@pytest.mark.parametrize("schema", SCHEMAS)
def test_translate_corpora(ctx, schema):
    total = {}
    for override, prefix, force in CONFIGS:
        if prefix is not None and schema != "openai":
            continue
        c = cfg(ctx, schema, override, prefix, force)
        for name, bodies in _translate_corpora().items():
            got = ctx.embeddings_translate_large(c, bodies)
            ref = ctx.chat_translate(c, bodies)
            n, esc = same_as_translate_pass(bodies, got, ref, (schema, name, override, prefix, force))
            total[name] = (total.get(name, (0, 0))[0] + n, total.get(name, (0, 0))[1] + esc)
    print("\n%s: compared with the translate pass (bodies, escaped-key declines) %s" % (schema, total))
    assert total["emb_body"][0] > 3000 and total["emb_body"][1] == 0


# ================================================================ 2. large realistic requests: every one OK, byte-exact
@pytest.mark.parametrize("schema", SCHEMAS)
@pytest.mark.parametrize("override", ["", "text-embedding-005"])
def test_large_realistic(ctx, schema, override):
    bodies = L.large_corpus()
    if schema == "aws-bedrock":
        bodies = [b for b in bodies if isinstance(json.loads(b)["input"], str)] + L.titan_bodies()
    elif schema == "gcp-vertexai":
        bodies = [b for b in bodies if not isinstance(json.loads(b)["input"][0] if isinstance(json.loads(b)["input"], list) else "", (int, list))]
    got = ctx.embeddings_translate_large(cfg(ctx, schema, override), bodies)
    check_oracle(schema, bodies, got, override)


# ================================================================ 3. features at the scan's boundaries
@pytest.mark.parametrize("schema", ["gcp-vertexai", "openai"])
def test_boundaries(ctx, schema):
    corpus = L.boundary_corpus()
    labels, bodies = [l for l, _ in corpus], [b for _, b in corpus]
    got = ctx.embeddings_translate_large(cfg(ctx, schema, "o-1"), bodies)
    for l, b, g in zip(labels, bodies, got):
        name = l.split()[0]
        t = O.embeddings_translate(schema, b, model_override="o-1")
        if name in L.OK_FEATURES or name in ("null_elem", "model") or (schema == "openai" and name in ("lone_high", "lone_low", "bs_u_literal")):
            assert g["status"] == OK == t.status, (l, g["reason"], t.err)
            assert g["body"] == t.body and g["path"].decode() == t.path, (l, g["body"][:100], t.body[:100])
        elif name == "number_elem" or name == "nested_elem":
            assert g["status"] == E400, (l, g)
        else:   # lone surrogates in a re-encoded string (an escaped backslash before "ud83d" leaves the low half alone), bad hex
            assert (g["status"], g["reason"]) == (DECLINED, R_ESCAPE), (l, g)


# ================================================================ 4. limits
def test_limits(ctx):
    c = cfg(ctx, "gcp-vertexai")
    head, tail = b'{"model":"m","input":["', b'"]}'
    fit = head + b"a" * ((16 << 20) - 1 - len(head) - len(tail)) + tail
    over = head + b"a" * ((16 << 20) - len(head) - len(tail)) + tail
    g = ctx.embeddings_translate_large(c, [fit, over])
    assert (g[0]["status"], g[1]["status"], g[1]["reason"]) == (OK, DECLINED, R_TOO_LARGE), (g[0]["reason"], g[1]["reason"])
    check_oracle("gcp-vertexai", [fit], g[:1])
    # tokens: len / 2 + 1024 (token ids cost two tokens each)
    oc = cfg(ctx, "openai")
    def ids(k, n):
        b = b'{"model":"m","input":[' + b",".join([b"7"] * k) + b"]}"
        return b + b" " * (n - len(b))
    n = 400000
    cap = n // 2 + 1024
    k = (cap - 8) // 2
    while E.count_tokens(ids(k + 1, n)) <= cap: k += 1
    while E.count_tokens(ids(k, n)) > cap: k -= 1
    a, b = ids(k, n), ids(k + 1, n)
    assert E.count_tokens(a) <= cap < E.count_tokens(b)
    g = ctx.embeddings_translate_large(oc, [a, b])
    assert (g[0]["status"], g[1]["status"], g[1]["reason"]) == (OK, DECLINED, R_TOKENS), (g[0]["reason"], g[1]["reason"])
    # depth 48 is OK, 49 declines
    deep = [b'{"model":"m","input":"a","x":' + b"[" * d + b"]" * d + b"}" for d in (47, 48)]
    assert [(x["status"], x["reason"]) for x in ctx.embeddings_translate_large(oc, deep)] == [(OK, 0), (DECLINED, R_DEPTH)]
    # a 1 MiB unknown nested member
    meta = json.dumps({"trace": [{"id": i, "tags": [None, True, "x" * 200, {"k": [1.5, -2, []]}]} for i in range(4500)]}).encode()
    big = b'{"model":"m","metadata":' + meta + b',"input":["a","b"]}'
    got = ctx.embeddings_translate_large(cfg(ctx, "gcp-vertexai", "o"), [big])
    check_oracle("gcp-vertexai", [big], got, "o")


def _ceiling_bodies():
    """a Vertex record exactly at the output ceiling (16 * len + 65536) and one byte over it, at the same body length"""
    N, task = 20001, "T" * 100
    def body(t, first, spaces):
        return b'{"model":"m","task_type":"' + (task + "U" * t).encode() + b'","input":[' + first + b"," + b",".join([b"null"] * (N - 1)) + b"]}" + b" " * spaces
    def rec(b):
        t = O.embeddings_translate("gcp-vertexai", b)
        assert t.status == O.OK, t.err
        return len(t.path) + len(t.body)
    for t in range(16):
        b0 = body(t, b'"a"', 0)
        r = rec(b0)
        if (r - 65536) % 16 == 0:
            s = (r - 65536) // 16 - len(b0)
            assert s > 0
            at, over = body(t, b'"a"', s), body(t, b'"ab"', s - 1)
            assert len(at) == len(over) and rec(at) == 16 * len(at) + 65536 and rec(over) == rec(at) + 1
            return at, over
    raise AssertionError("no length residue found")


def test_output_ceiling(ctx):
    at, over = _ceiling_bodies()
    g = ctx.embeddings_translate_large(cfg(ctx, "gcp-vertexai"), [at, over])
    assert g[0]["status"] == OK and (g[1]["status"], g[1]["reason"]) == (DECLINED, R_OUT_SPACE), (g[0]["reason"], g[1]["reason"])
    check_oracle("gcp-vertexai", [at], g[:1])


def test_record_beyond_4gib(ctx):
    """a request-level task_type repeated for every null input: under 1 MB of body asks for tens of GB of record, more than 2^32
    bytes; the record's length must not wrap below the ceiling"""
    for t_len, n in ((524911, 90000), (300000, 14400), (65536, 65600)):
        body = b'{"task_type":"' + b"T" * t_len + b'","input":[""' + b",null" * (n - 1) + b"]}"
        assert len(body) < 1 << 20 and n * t_len > 1 << 32
        c = cfg(ctx, "gcp-vertexai")
        got, res = device_translate(ctx, c, [body], out_cap=1 << 26)
        host = ctx.embeddings_translate_large(c, [body])
        for g in (got[0], host[0]):
            assert (g["status"], g["reason"]) == (DECLINED, R_OUT_SPACE), (t_len, n, g)
        assert int(res[0]["body_len"]) == 0


# ================================================================ 5. the device form, 6. call composition
def device_translate(ctx, c, bodies, out_cap):
    import aigw_b200 as A
    from aigw_b200 import capi
    arena, offs, lens = A.pack_bodies(bodies)
    n = len(bodies)
    d_b, d_o, d_l, d_out, d_r, d_u = (ctx.dalloc(max(16, x)) for x in (arena.nbytes, offs.nbytes, lens.nbytes, out_cap, n * 32, 8))
    try:
        ctx.h2d(d_b, arena); ctx.h2d(d_o, offs); ctx.h2d(d_l, lens); ctx.memset(d_u, 0, 8)
        ctx.embeddings_translate_large_device(c, d_b, d_o, d_l, n, int(lens.max()), d_out, out_cap, d_r, d_u)
        ctx.sync()
        res = np.zeros(n, dtype=capi.DocResult); used = np.zeros(1, dtype=np.uint64)
        ctx.d2h(res, d_r); ctx.d2h(used, d_u)
        out = np.zeros(max(16, min(int(used[0]), out_cap)), dtype=np.uint8)
        ctx.d2h(out, d_out, min(int(used[0]), out_cap))
    finally:
        for d in (d_b, d_o, d_l, d_out, d_r, d_u):
            ctx.dfree(d)
    return ctx._records(bodies, res, out), res


def test_out_space_and_host_retry(ctx):
    bodies = [b for b in L.large_corpus() if isinstance(json.loads(b)["input"], str) or isinstance(json.loads(b)["input"][0], (str, dict))][:12]
    c = cfg(ctx, "gcp-vertexai", "text-embedding-005")
    got, res = device_translate(ctx, c, bodies, out_cap=sum(len(b) for b in bodies) // 3)
    host = ctx.embeddings_translate_large(c, bodies)
    fit = [i for i, g in enumerate(got) if g["status"] == OK]
    assert fit and len(fit) < len(bodies)
    for i, g in enumerate(got):
        if g["status"] != OK:
            assert (g["status"], g["reason"]) == (DECLINED, R_OUT_SPACE)
            assert int(res[i]["body_len"]) == len(host[i]["path"]) + len(host[i]["body"])   # the record length it needs
        else:
            assert all(g[k] == host[i][k] for k in KEYS)
    check_oracle("gcp-vertexai", bodies, host, "text-embedding-005")
    # a record far above the host form's first arena (2 * len + 1024): the retry takes it
    at, _ = _ceiling_bodies()
    check_oracle("gcp-vertexai", [at], ctx.embeddings_translate_large(cfg(ctx, "gcp-vertexai"), [at]))


def test_composition_and_device_form(ctx):
    r = random.Random(5)
    rng = np.random.default_rng(7)
    mixed = L.large_corpus(total=6 << 20) + [EG.emb_body(rng) for _ in range(200)] + EG.ODD + [b for _, b in L.boundary_corpus()][::9]
    r.shuffle(mixed)
    for schema in ("gcp-vertexai", "openai"):
        c = cfg(ctx, schema, "m2")
        whole = ctx.embeddings_translate_large(c, mixed)
        order = list(range(len(mixed)))
        r.shuffle(order)
        rev = ctx.embeddings_translate_large(c, [mixed[i] for i in order])
        cut = len(mixed) // 3
        split = ctx.embeddings_translate_large(c, mixed[:cut]) + ctx.embeddings_translate_large(c, mixed[cut:])
        dev, _ = device_translate(ctx, c, mixed, sum(2 * len(b) + 2048 for b in mixed))
        for j, i in enumerate(order):
            assert all(rev[j][k] == whole[i][k] for k in KEYS), i
        for i in range(len(mixed)):
            assert all(split[i][k] == whole[i][k] for k in KEYS), i
            assert all(dev[i][k] == whole[i][k] for k in KEYS), i


def test_other_schemas_decline(ctx):
    body = b'{"model":"m","input":"a"}'
    for schema in (0, 1, 3, 512, 519, 7, 64, 36):
        g = ctx.embeddings_translate_large(ctx.cfg(schema), [body, body + b" " * 100000])
        assert [(x["status"], x["reason"]) for x in g] == [(DECLINED, R_SCHEMA)] * 2, schema
