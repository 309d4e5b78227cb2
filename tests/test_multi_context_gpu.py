"""Several contexts in one process (ADVICE r1: per-device one-time setup, cudaSetDevice at every entry point): two contexts on one GPU driven
from two threads at once — the bench's --e2e-lanes mode and a gateway with several worker threads do exactly this — and, when the box has a
second GPU, one context per device.  Every result is checked against the oracle."""
import threading

import numpy as np
import pytest

import _oracle as O
import _workload as W

pytestmark = pytest.mark.gpu


def _bodies(seed, n):
    arena, offs, lens = W.chat_corpus(2, seed, n)
    return [bytes(arena[int(offs[i]):int(offs[i]) + int(lens[i])]) for i in range(n)]


def _check(ctx, bodies, errors, rounds=3):
    import aigw_b200 as A
    try:
        exp = [O.chat_translate("aws-bedrock", b) for b in bodies]
        for _ in range(rounds):
            got = ctx.chat_translate(ctx.cfg("aws-bedrock"), bodies)
            for g, o in zip(got, exp):
                assert g["status"] == A.AIGW_OK and o.status == O.OK and g["body"] == o.body and g["path"].decode() == o.path
            (h,) = ctx.stream_open("openai", b"req-model")
            r = ctx.stream_chunk(h, b'data: {"model":"m","usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}\n\n', True)
            assert r["status"] == 0 and r["usage"] == (3, -1, -1, 4, 7, -1) and r["model"] == b"m"
            ctx.stream_close([h])
    except BaseException as e:   # noqa: BLE001 - reported by the main thread
        errors.append(e)


def test_two_contexts_one_device_two_threads():
    import aigw_b200 as A
    c1, c2 = A.Context(0), A.Context(0)
    try:
        errors = []
        ts = [threading.Thread(target=_check, args=(c1, _bodies(1, 3000), errors)), threading.Thread(target=_check, args=(c2, _bodies(2, 700), errors))]
        for t in ts: t.start()
        for t in ts: t.join()
        assert not errors, errors[0]
    finally:
        c1.close(); c2.close()


def test_one_context_per_device():
    import aigw_b200 as A
    try:
        c1 = A.Context(1)
    except Exception:   # noqa: BLE001
        pytest.skip("the box has one GPU")
    c0 = A.Context(0)
    try:
        errors = []
        ts = [threading.Thread(target=_check, args=(c0, _bodies(3, 2000), errors)), threading.Thread(target=_check, args=(c1, _bodies(4, 2000), errors))]
        for t in ts: t.start()
        for t in ts: t.join()
        assert not errors, errors[0]
        _check_device_call_on_other_device(c0, c1)
    finally:
        c0.close(); c1.close()


def _check_device_call_on_other_device(c0, c1):
    """A device-buffer call of c1 made while this thread's current device is c0's still runs on c1's GPU."""
    import aigw_b200 as A
    n = 64
    buf, coff, cfirst = W.sse_corpus(4, 0, n)
    d = [c1.dalloc(a.nbytes) for a in (buf, coff, cfirst)] + [c1.dalloc(n * A.SseResult.itemsize)]
    try:
        for p, a in zip(d, (buf, coff, cfirst)):
            c1.h2d(p, a)
        c0.sync()   # makes c0's device current
        c1.sse_usage_device(d[0], d[1], d[2], n, d[3])
        res = np.zeros(n, dtype=A.SseResult)
        c1.d2h(res, d[3])
    finally:
        for p in d:
            c1.dfree(p)
    raw = bytes(buf)
    for s in range(n):
        st = O.SSEStream(); acc = [-1] * 6
        for c in range(int(cfirst[s]), int(cfirst[s + 1])):
            u = st.feed(raw[int(coff[c]):int(coff[c + 1])]).as_tuple()
            acc = [v if v >= 0 else a for a, v in zip(acc, u)]
        r = res[s]; m = int(r["mask"])
        got = [int(r["input"]) if m & 1 else -1, int(r["cached"]) if m & 8 else -1, int(r["cache_creation"]) if m & 16 else -1,
               int(r["output"]) if m & 2 else -1, int(r["total"]) if m & 4 else -1, int(r["reasoning"]) if m & 32 else -1]
        assert int(r["status"]) == 0 and got == acc, s
