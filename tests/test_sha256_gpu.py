"""SigV4 payload hash on the GPU (internal/backendauth/aws.go:93-117): FIPS 180-4 known answers, hashlib / oracle parity, translate-record bodies."""
import hashlib

import numpy as np
import pytest

import _oracle as O
import _workload as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gw():
    from aigw_b200 import capi
    g = capi.Context(0)
    yield g
    g.close()


def pack(msgs, align=1, lead=0):
    offs, pos = [], lead
    for m in msgs:
        pos = (pos + align - 1) // align * align
        offs.append(pos); pos += len(m)
    arena = np.zeros(pos + 64, dtype=np.uint8)
    for o, m in zip(offs, msgs):
        arena[o:o + len(m)] = np.frombuffer(m, dtype=np.uint8)
    return arena, np.array(offs, dtype=np.uint64), np.array([len(m) for m in msgs], dtype=np.uint32)


def test_known_answers_and_boundaries(gw):
    kat = [b"abc", b"", b"abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq",
           b"abcdefghbcdefghicdefghijdefghijkefghijklfghijklmghijklmnhijklmnoijklmnopjklmnopqklmnopqrlmnopqrsmnopqrstnopqrstu", b"a" * 1000000]
    rng = np.random.default_rng(1)
    msgs = kat + [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in list(range(0, 200)) + [4095, 4096, 4097, 65535, 65536, 100003]]
    for align, lead in [(1, 0), (1, 1), (1, 2), (1, 3), (16, 0), (4, 0)]:   # every start alignment
        arena, offs, lens = pack(msgs, align, lead)
        dig = gw.sha256_host(arena, offs, lens)
        for m, d in zip(msgs, dig):
            assert bytes(d) == hashlib.sha256(m).digest()
    assert bytes(dig[0]).hex() == "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad"
    assert bytes(dig[0]) == O.sha256(b"abc")


def test_translate_record_bodies(gw):
    """digest of every Bedrock body the translate pass produced, straight from its output arena"""
    from aigw_b200 import capi
    n = 20000
    arena, offs, lens = W.chat_corpus(2, 0, n)
    bodies = [bytes(arena[int(offs[i]):int(offs[i]) + int(lens[i])]) for i in range(n)]
    bodies[7] = b'{"model":5}'   # a 400: zero digest
    arena, offs, lens = capi.pack_bodies(bodies)
    cfg = capi.Context.cfg("aws-bedrock")
    out_cap = 2 * len(arena) + 600 * n
    d_b = gw.dalloc(len(arena) + 64); d_o = gw.dalloc(offs.nbytes); d_l = gw.dalloc(lens.nbytes); d_out = gw.dalloc(out_cap); d_r = gw.dalloc(n * 32); d_u = gw.dalloc(64); d_d = gw.dalloc(n * 32)
    gw.h2d(d_b, arena); gw.h2d(d_o, offs[:n].copy()); gw.h2d(d_l, lens); gw.memset(d_u, 0, 8)
    gw.chat_translate_device(cfg, d_b, d_o, d_l, n, int(lens.max()), d_out, out_cap, d_r, d_u)
    gw.chat_body_sha256_device(d_out, d_r, n, d_d)
    res = np.zeros(n, dtype=capi.DocResult); gw.d2h(res, d_r)
    dig = np.zeros((n, 32), dtype=np.uint8); gw.d2h(dig, d_d)
    used = np.zeros(1, dtype=np.uint64); gw.d2h(used, d_u)
    out = np.zeros(int(used[0]), dtype=np.uint8); gw.d2h(out, d_out, int(used[0]))
    assert res[7]["status"] == 1 and not dig[7].any()
    for i in list(range(0, n, 97)) + [8, 9]:
        if i == 7: continue
        r = res[i]; o = int(r["out_off"]) + int(r["path_len"])
        body = bytes(out[o:o + int(r["body_len"])])
        assert r["status"] == 0 and bytes(dig[i]) == hashlib.sha256(body).digest()
    for p in (d_b, d_o, d_l, d_out, d_r, d_u, d_d): gw.dfree(p)


def test_translate_host_after_larger_hash_host():
    """a larger hash host call leaves the translate pipeline's chunk slots alone: a translate call after it on a fresh context still
    gets a result table for its own batch"""
    from aigw_b200 import capi
    c = capi.Context(0)
    try:
        arena, offs, lens = W.chat_corpus(2, 0, 1200)
        bodies = [bytes(arena[int(offs[i]):int(offs[i]) + int(lens[i])]) for i in range(1200)]
        dig = c.sha256_host(arena, offs, lens)
        assert all(bytes(dig[i]) == hashlib.sha256(bodies[i]).digest() for i in range(0, 1200, 50))
        c.chat_set_small_batch(0)   # the throughput pipeline, which uses the chunk slots
        got = c.chat_translate(c.cfg("aws-bedrock"), bodies[:1000])
        for b, g in zip(bodies, got):
            o = O.chat_translate("aws-bedrock", b)
            assert g["status"] == 0 and o.status == O.OK and g["body"] == o.body and g["path"].decode() == o.path
    finally:
        c.close()
