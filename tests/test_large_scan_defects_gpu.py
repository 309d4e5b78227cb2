"""The malformed corpora of test_large_scan_defects_cpu.py (probe mutations, truncations, backslash runs, bodies of 16 MiB - 1)
through aigw_{chat,embeddings,rerank}_translate_large_host, each body against the oracle under a few configurations:
  * an OK is an oracle OK with the same ":path", body bytes, body kind, model span, stream flag and flags;
  * a 400 (422, 500) is the oracle's 400 (422, 500);
  * an oracle 400 is a GPU 400 when the scan has no excuse to decline: the defect neither writes nor removes a backslash or an
    escaped byte, and by scan_model the body has no control byte or invalid escape inside a string and no key holding an escape;
  * an oracle OK the scan has no such excuse to decline is a GPU OK, or a capacity decline (tokens, ops, scratch, depth), a
    non-canonical number in chat's tool parameters, or a repeated key;
  * any other decline carries a reason the kernel documents (include/aigw_b200.h), tallied and printed per reason.
Bodies of at most 64 KiB also give the translate pass's answer.  Then the whole corpus, interleaved with valid large requests, in
one call, in reverse order and split across two calls: every answer is the one the body had alone in its corpus call (the CTAs
are persistent and pull requests from a counter, so this catches state a rejected request leaves to the next one)."""
import json
import time

import pytest

import _oracle as O
import test_chat_large_cpu as CL
import test_chat_large_gpu as CG
import test_embeddings_large_cpu as EL
import test_embeddings_large_gpu as EGL
import test_large_scan_defects_cpu as D
import test_rerank_large_cpu as RL
import test_rerank_large_gpu as RGL

pytestmark = pytest.mark.gpu

OK, E400, E422, E500, DECLINED = 0, 1, 2, 3, 4
R_CTRL, R_ESCAPE, R_TOKENS, R_OPS, R_SCRATCH, R_DUP_KEY, R_UNSUPPORTED, R_NUMBER, R_CONTENT, R_TOOL, R_DEPTH, R_ROOT = 3, 4, 5, 6, 7, 9, 11, 12, 14, 15, 16, 17
# the declines each call documents for bodies below 16 MiB in the host form: its own (escapes, capacities, depth) and those of
# the translate pass whose results it gives
DECLINES = {
    "chat": {R_CTRL, R_ESCAPE, R_TOKENS, R_OPS, R_SCRATCH, R_DUP_KEY, R_UNSUPPORTED, R_NUMBER, R_CONTENT, R_TOOL, R_DEPTH, R_ROOT},
    "emb": {R_CTRL, R_ESCAPE, R_TOKENS, R_OPS, R_SCRATCH, R_DUP_KEY, R_UNSUPPORTED, R_NUMBER, R_DEPTH},
    "rerank": {R_CTRL, R_ESCAPE, R_TOKENS, R_DUP_KEY, R_UNSUPPORTED, R_DEPTH, R_ROOT},
}
CONFIGS = {
    "chat": [("openai", "ovr-model", True, False), ("azure-openai", None, False, False), ("openai", None, False, True)],
    "emb": [(s, ov, False, False) for s in EGL.SCHEMAS for ov in ("", "text-embedding-005")],
    "rerank": [("rerank", "", False, False), ("rerank", "rerank-v3.5", False, False), ("rerank", "", False, True)],
}
HOST = {"chat": "chat_translate_large_host", "emb": "embeddings_translate_large_host", "rerank": "rerank_translate_large_host"}
KEYS = ("status", "reason", "path", "body", "body_kind", "model", "stream", "flags")
VERSION = CG.VERSION


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def make_cfg(ctx, kernel, conf):
    schema, ov, cost, force = conf
    if kernel == "chat":
        return CG.cfg(ctx, schema, ov, cost, force)
    if kernel == "emb":
        return EGL.cfg(ctx, schema, ov, force=force)
    return RGL.cfg(ctx, ov, force=force)


def call(ctx, kernel, c, bodies):
    import aigw_b200 as A
    arena, offs, lens = A.pack_bodies(bodies)
    res, out, _ = getattr(ctx, HOST[kernel])(c, arena, offs, lens)
    recs = ctx._records(bodies, res, out)
    for r, x in zip(recs, res):
        r["flags"] = int(x["flags"])
    return recs


def oracle(kernel, conf, body):
    """(status, record fields an OK must match or None)"""
    schema, ov, cost, force = conf
    if kernel == "chat":
        t = O.chat_translate(schema, body, model_override=ov or "", cost_configured=cost, force=force, prefix=VERSION if schema == "azure-openai" else "v1")
        if t.status != O.OK:
            return t.status, None
        forced = False
        if cost and t.stream:
            so = json.loads(body.decode("utf-8", "replace"), strict=False).get("stream_options")   # raw control bytes are the decoder's default
            forced = not (isinstance(so, dict) and so.get("include_usage") is True)
        return OK, {"path": t.path.encode(), "body": t.body if t.body_kind == O.BYTES else b"", "body_kind": t.body_kind, "model": t.model,
                    "stream": t.stream, "flags": int(t.stream) | (2 if forced else 0)}
    if kernel == "emb":
        t = O.embeddings_translate(schema, body, model_override=ov, prefix=VERSION if schema == "azure-openai" else "v1", force=force)
        if t.status != O.OK:
            return t.status, None
        return OK, {"path": t.path.encode(), "body": t.body if t.body_kind == O.BYTES else b"", "body_kind": t.body_kind, "model": t.model,
                    "stream": False, "flags": 0}
    v, path, out, model = RGL.expect(body, ov, "v2", force)
    if v != RGL.Q.OK:
        return (E400 if v == RGL.Q.FAIL else DECLINED), None
    return OK, {"path": path.encode(), "body": out or b"", "body_kind": 0 if out is None else 1, "model": model, "stream": False, "flags": 0}


_FLAGS = {}


def flags(kernel, label, body):
    """D.scan_flags, once per body"""
    if (kernel, label) not in _FLAGS:
        _FLAGS[(kernel, label)] = D.scan_flags(body)
    return _FLAGS[(kernel, label)]


def no_excuse(kernel, label, at, body):
    """an oracle 400 the GPU must answer with 400: the defect leaves every backslash and escaped byte as it was (the runs: their
    defect is the parity), and the scan itself has nothing to decline for"""
    return not D.defect_touches_escape(kernel, label, at) and not flags(kernel, label, body)


def _dup_key(pairs):
    if len({k for k, _ in pairs}) != len(pairs):
        raise KeyError("repeated key")
    return dict(pairs)


def repeated_key(body):
    try:
        json.loads(body.decode("utf-8", "replace"), strict=False, object_pairs_hook=_dup_key)
    except KeyError:
        return True
    except ValueError:
        pass
    return False


def ok_decline_explained(kernel, label, body, reason):
    """a decline of a body the oracle accepts: the scan's own reasons (a control byte in a string, an escape, an escaped key),
    or a capacity, or a rule of the translate pass the decoder does not have"""
    if flags(kernel, label, body):
        return True
    if reason in (R_TOKENS, R_OPS, R_SCRATCH, R_DEPTH):
        return True
    if kernel == "chat" and reason == R_NUMBER:   # tool parameters are re-printed: a non-canonical number declines
        return True
    return reason == R_DUP_KEY and repeated_key(body)


def check(kernel, conf, corpus, got, tally, bad):
    """the per-body contract; violations go to `bad`, the (status, reason) split to `tally`"""
    for (label, bound, at, body), g in zip(corpus, got):
        st, want = oracle(kernel, conf, body)
        where = (kernel, conf, label, len(body), (g["status"], g["reason"]), st)
        key = ("ok",) if g["status"] == OK else ("400",) if g["status"] == E400 else (g["status"], g["reason"])
        tally[key] = tally.get(key, 0) + 1
        if g["status"] == OK:
            if st != OK:
                bad.append(where + ("GPU OK, oracle not",))
            elif any(g[k] != want[k] for k in want):
                bad.append(where + ({k: (g[k][:80] if isinstance(g[k], bytes) else g[k], want[k][:80] if isinstance(want[k], bytes) else want[k])
                                     for k in want if g[k] != want[k]},))
        elif g["status"] in (E400, E422, E500):
            if st != g["status"]:
                bad.append(where + ("GPU error status, oracle not the same",))
        elif g["status"] != DECLINED:
            bad.append(where + ("unknown status",))
        elif g["reason"] not in DECLINES[kernel]:
            bad.append(where + ("undocumented decline",))
        elif st == E400 and no_excuse(kernel, label, at, body):
            bad.append(where + ("oracle 400 with no excuse to decline",))
        elif st == OK and not ok_decline_explained(kernel, label, body, g["reason"]):
            bad.append(where + ("oracle OK with no excuse to decline",))


def same_as_translate_pass(kernel, ctx, c, corpus, got):
    """bodies of at most 64 KiB: the translate pass's answer (its capacity declines skipped; the large call's documented extra
    declines counted).  Returns (compared, extra declines)."""
    idx = [i for i, (_, _, _, b) in enumerate(corpus) if len(b) <= 65536]
    bodies = [corpus[i][3] for i in idx]
    ref = ctx.chat_translate(c, bodies)
    g = [got[i] for i in idx]
    if kernel == "emb":
        return EGL.same_as_translate_pass(bodies, g, ref, "defects")
    compared = extra = 0
    for i, b, x, h in zip(idx, bodies, g, ref):
        if h["status"] == DECLINED and h["reason"] in (1, R_TOKENS, R_OPS, R_SCRATCH, 18):
            continue
        if kernel == "chat" and x["status"] == DECLINED and h["status"] != DECLINED:
            # documented: a key with a backslash anywhere, a lone surrogate anywhere (the corpus holds no \u escape in chat)
            assert x["reason"] == R_ESCAPE and "escaped_key" in flags(kernel, corpus[i][0], b), (corpus[i][0], x["reason"], h["status"], h["reason"])
            extra += 1
            continue
        keys = ("status", "path", "body", "body_kind", "model", "stream")
        assert all(x[k] == h[k] for k in keys), (kernel, corpus[i][0], {k: (x[k], h[k]) for k in keys if x[k] != h[k]}, x["reason"], h["reason"])
        compared += 1
    return compared, extra


_ANSWERS = {}


def corpus_answers(ctx, kernel, conf):
    """the defect corpus in one call under conf (cached for the composition test)"""
    key = (kernel, conf)
    if key not in _ANSWERS:
        corpus = D.defect_corpus(kernel)
        _ANSWERS[key] = call(ctx, kernel, make_cfg(ctx, kernel, conf), [b for *_, b in corpus])
    return _ANSWERS[key]


@pytest.mark.parametrize("kernel", D.KERNELS)
def test_defects_against_oracle(ctx, kernel):
    t0 = time.time()
    corpus = D.defect_corpus(kernel)
    near = D.near_limit_corpus(kernel)
    if kernel == "rerank":
        RL.verdicts([b for *_, b in corpus + near])
    bad = []
    print("\n%s: %d bodies, %.1f MB (+ %d of 16 MiB - 1)" % (kernel, len(corpus), sum(len(b) for *_, b in corpus) / 1e6, len(near)))
    for conf in CONFIGS[kernel]:
        tally = {}
        got = corpus_answers(ctx, kernel, conf)
        check(kernel, conf, corpus, got, tally, bad)
        # the bodies of 16 MiB - 1 in a call of their own: their workspace slices leave room for few CTAs
        check(kernel, conf, near, call(ctx, kernel, make_cfg(ctx, kernel, conf), [b for *_, b in near]), tally, bad)
        n, extra = same_as_translate_pass(kernel, ctx, make_cfg(ctx, kernel, conf), corpus, got)
        print("  %s: GPU (status or (status, reason)) %s; %d compared with the translate pass, %d documented extra declines"
              % (conf, dict(sorted(tally.items(), key=str)), n, extra))
    ost = {}
    for *_, b in corpus:
        s = oracle(kernel, CONFIGS[kernel][0], b)[0]
        ost[s] = ost.get(s, 0) + 1
    print("  oracle under %s: %s (0 OK, 1 400, 2 422, 3 500, 4 outside)" % (CONFIGS[kernel][0], ost))
    strict = sum(oracle(kernel, CONFIGS[kernel][0], b)[0] == E400 and no_excuse(kernel, l, at, b) for l, _, at, b in corpus + near)
    print("  %d oracle-400 bodies the GPU must answer with 400 (no escape touched, nothing for the scan to decline)" % strict)
    for x in bad[:30]:
        print("  VIOLATION", x)
    print("  %d violations, %.0f s" % (len(bad), time.time() - t0))
    assert not bad, bad[:5]


def _valid_large(kernel):
    if kernel == "chat":
        return [CL.long_chat(60 + i, 70000 + 90000 * i, CL.STREAM_MODES[i % 9]) for i in range(8)]
    if kernel == "emb":
        return EL.large_corpus(total=3 << 20)
    return list(RL.large_corpus()[4:16])


@pytest.mark.parametrize("kernel", D.KERNELS)
def test_composition(ctx, kernel):
    conf = CONFIGS[kernel][0]
    c = make_cfg(ctx, kernel, conf)
    corpus = [b for *_, b in D.defect_corpus(kernel)]
    alone = corpus_answers(ctx, kernel, conf)
    valid = _valid_large(kernel)
    valid_alone = call(ctx, kernel, c, valid)
    assert all(v["status"] == OK for v in valid_alone), [(v["status"], v["reason"]) for v in valid_alone]
    # the valid requests spread through the defects
    mixed, want = [], []
    step = len(corpus) // len(valid) + 1
    for i in range(0, len(corpus), step):
        j = i // step
        mixed += corpus[i:i + step] + valid[j:j + 1]
        want += alone[i:i + step] + valid_alone[j:j + 1]
    assert len(mixed) == len(corpus) + len(valid)
    whole = call(ctx, kernel, c, mixed)
    rev = call(ctx, kernel, c, mixed[::-1])[::-1]
    cut = len(mixed) // 3
    split = call(ctx, kernel, c, mixed[:cut]) + call(ctx, kernel, c, mixed[cut:])
    for name, got in (("one call", whole), ("reversed", rev), ("two calls", split)):
        diff = [i for i, (g, w) in enumerate(zip(got, want)) if any(g[k] != w[k] for k in KEYS)]
        assert not diff, (kernel, name, len(diff), [(len(mixed[i]), (got[i]["status"], got[i]["reason"]), (want[i]["status"], want[i]["reason"])) for i in diff[:5]])
    print("\n%s: %d requests in one call, reversed and in two calls give the answers they had alone" % (kernel, len(mixed)))
