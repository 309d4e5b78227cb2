"""Corpora of Cohere /v2/rerank requests for aigw_rerank_translate_large_* (test_rerank_large_gpu.py feeds them through the GPU),
and the CPU checks of those corpora: the generators are deterministic by seed, and the oracle (tests/_rerank_oracle.py) agrees
with json.loads wherever both apply.

  large realistic   RAG reranks of 64 KiB to 8 MiB: a query plus 50-5 000 retrieved chunks of 200-4 000 characters, built from
                    test_rerank_cpu's WORDS (escapes, non-ASCII, astral characters) with ensure_ascii / indent variants and the
                    UNKNOWN members (nested metadata, rank_fields); about 80 MB in all
  near the limit    bodies of 16 MiB - 1 and a little less (accepted) and of exactly 16 MiB (AIGW_R_TOO_LARGE)
  boundaries        each feature (backslash runs before a quote, \\u escapes, string starts and ends, null and number elements,
                    the model member, invalid escapes) at every offset within +-40 bytes of a thread (32 B), warp (1 KiB) and
                    tile (8 KiB) boundary of the scan; body lengths k * 8192 +- 1
  splices           where the model override goes: the model last after megabytes of documents, no model (white space around
                    the root, an empty root), a null model, the model twice"""
import functools
import hashlib
import json
import math
import multiprocessing
import os
import random

import _rerank_oracle as Q
import test_rerank_cpu as G

MIB = 1 << 20
LIMIT = 16 * MIB          # bodies of this size and above are AIGW_R_TOO_LARGE
THREAD, WARP, TILE = 32, 1024, 8192
# boundaries of each kind inside the first two tiles, away from the others: byte 3200 starts a thread (not a warp), 5120 a warp
# (not a tile), 8192 a tile
BOUNDS = (("thread", 3200), ("warp", 5120), ("tile", 8192))
OFFSETS = range(-40, 41)


# ================================================================ large realistic requests
def _pool(r, n=60000):
    return " ".join(r.choice(G.WORDS) for _ in range(n))


def large_request(seed, target):
    """one RAG rerank of about `target` bytes (at least 64 KiB + 1)"""
    r = random.Random(seed)
    pool = _pool(r)
    chars = target / 1.3   # characters: UTF-8, \u escapes and indentation make the bytes more
    n = int(min(5000, max(50, chars / r.uniform(600, 2500))))
    mean = min(4000, max(200, chars / n))

    def chunk():
        ln = int(min(4000, max(200, mean * r.uniform(0.5, 1.5))))
        o = r.randrange(len(pool) - ln)
        return pool[o:o + ln]

    req = {"model": r.choice(G.MODELS), "query": chunk()[:r.randint(5, 200)], "documents": [chunk() for _ in range(n)]}
    if r.random() < 0.6:
        req["top_n"] = r.randint(1, n)
    if r.random() < 0.3:
        req["max_tokens_per_doc"] = r.choice((512, 1024, 4096))
    if r.random() < 0.4:
        for k in r.sample(sorted(G.UNKNOWN), r.randint(1, 3)):
            req[k] = G.UNKNOWN[k](r)
    keys = list(req)
    r.shuffle(keys)
    req = {k: req[k] for k in keys}
    body = json.dumps(req, ensure_ascii=r.random() < 0.3, indent=2 if r.random() < 0.2 else None,
                      separators=None if r.random() < 0.5 else (",", ":")).encode()
    if len(body) <= 65536:
        return large_request(seed + 7919, target * 1.5)
    return body if len(body) <= 8 * MIB else large_request(seed + 7919, target * 0.8)


@functools.lru_cache(maxsize=None)
def large_corpus(n=300, seed=41):
    """n bodies from 64 KiB to 8 MiB: four large ones (1, 2, 4 and 8 MiB), the rest log-normal around 150 KB"""
    r = random.Random(seed)
    out = []
    for i in range(n):
        target = (MIB, 2 * MIB, 4 * MIB, 8 * MIB - 65536)[i] if i < 4 else min(MIB, max(65537, r.lognormvariate(math.log(150000), 0.6)))
        out.append(large_request(seed * 1000003 + i, target))
    return out


def sized_body(length, seed=5):
    """a realistic rerank of exactly `length` bytes: documents from the pool, the last one ASCII letters padded to fit"""
    r = random.Random(seed)
    pool = _pool(r)
    head = b'{"model":"rerank-v3.5","query":"what is the refund policy","documents":['
    parts, size = [], len(head) + 2
    while size < length - 70000:
        o = r.randrange(len(pool) - 4000)
        d = json.dumps(pool[o:o + r.randint(200, 4000)], ensure_ascii=False).encode() + b","
        parts.append(d)
        size += len(d)
    pad = length - size - 2
    assert pad > 0
    letters = bytes(r.choice(b"abcdefghij klmnop") for _ in range(pad))
    body = head + b"".join(parts) + b'"' + letters + b'"]}'
    assert len(body) == length
    return body


@functools.lru_cache(maxsize=None)
def near_limit_bodies():
    """(body, accepted): 16 MiB - 1, - 100, - 8192 - 1 are accepted, 16 MiB is not"""
    return [(sized_body(LIMIT - d, seed=d), True) for d in (1, 100, 8193)] + [(sized_body(LIMIT, seed=0), False)]


# ================================================================ features at the scan's thread, warp and tile boundaries
HEAD = b'{"query":"'
OPEN = b'","documents":["x","'   # closes the query string, opens the documents array and a document string


def _place(at, pre, feat, post, length):
    """HEAD + query text + pre + feat + post + document text + '"]}', with byte `at` of the body at the start of feat and
    `length` bytes in all; every post leaves the scan inside a document string, whose text pads the body"""
    body = HEAD + b"q" * (at - len(HEAD) - len(pre)) + pre + feat + post
    body += b"d" * (length - len(body) - 3) + b'"]}'
    assert len(body) == length and body[at:at + len(feat)] == feat, (len(body), length)
    return body


def _features():
    """name -> (pre, feat, post), starting inside the query string"""
    return {
        "u_escape": (b"", b"\\u00e9\\uD83D\\uDE00", OPEN),
        "u_bad": (b"", b"\\u12G4", OPEN),
        "bad_escape": (b"", b"\\q", OPEN),
        "string_start": (OPEN[:-1], b'"doc', b'","'),
        "string_end": (OPEN + b"doc", b'"', b',"'),
        "null_elem": (OPEN[:-1], b"null", b',"'),
        "number_elem": (OPEN[:-1], b"123", b',"'),
        "model": (b'","model":', b'"rerank-v3.5"', b',"documents":["x","'),
    }


def _run(n):
    """n backslashes and a quote: an odd run escapes the quote (the query string goes on), an even one leaves it closing"""
    return b"", b"\\" * n + b'"', OPEN if n % 2 else OPEN[1:]


def boundary_corpus():
    """(label, body): every feature at every offset within +-40 bytes of each boundary kind, lengths k * 8192 +- 1; backslash
    runs of 1, 32, 33 and 64 before a quote at every offset, and, cycling over the placements, every length 1-70"""
    out = []
    idx = 0
    for kind, b in BOUNDS:
        for d in OFFSETS:
            at = b + d
            length = (TILE if b < TILE else 2 * TILE) + (1 if (d + b) % 2 else -1)
            for name, (pre, feat, post) in _features().items():
                out.append(("%s %s@%+d" % (name, kind, d), _place(at, pre, feat, post, length)))
            for n in sorted({1, 32, 33, 64, 1 + idx % 70}):
                out.append(("run%d %s@%+d" % (n, kind, d), _place(at - n, *_run(n), length)))   # the quote on the boundary
            idx += 1
    for length in (TILE - 1, TILE + 1, 2 * TILE - 1, 2 * TILE + 1):   # a trailing backslash at the end of the body
        body = b'{"documents":["' + b"t" * (length - 16) + b"\\"
        assert len(body) == length
        out.append(("trailing backslash len %d" % length, body))
    return out


# ================================================================ splices of the model override
def splice_corpus():
    r = random.Random(9)
    pool = _pool(r, 20000)
    step = (len(pool) - 1500) // 97
    docs = [pool[(i % 97) * step:(i % 97) * step + 1500] for i in range(2100)]
    big = json.dumps(docs, ensure_ascii=False).encode()
    return [
        b'{"query":"q","documents":' + big + b',"top_n":3,"model":"rerank-v3.5"}',   # the model last, after megabytes
        b'{"query":"q","documents":' + big + b',"model":null}',
        b' \n\t{"query":"q","documents":' + big + b'} \r\n ',                          # no model, white space around the root
        b'{"documents":' + big + b'}',
        b"{}", b" { } ", b"\n{}\n", b'{"model":null}', b' {"model" : null , "query":"q"} ',
        b'{"model":"a","documents":' + big + b',"model":"b"}',                        # twice: declined
        b'{"model":"a","model":"b"}', b'{"documents":["a"],"metadata":{"model":"x"},"rank_fields":["model"]}',
    ]


# ================================================================ oracle verdicts, cached per body
@functools.lru_cache(maxsize=None)
def _key(body):
    return hashlib.sha1(body).digest()


_VERDICTS = {}


def _verdict(body):
    return Q.parse_body(body)


def verdicts(bodies):
    """Q.parse_body of every body, computed once per body (a few processes share the work: the oracle runs at about 2 MB/s)"""
    todo = [b for b in dict.fromkeys(bodies) if _key(b) not in _VERDICTS]
    if todo:
        if sum(len(b) for b in todo) > 4 * MIB and (os.cpu_count() or 1) > 1:
            with multiprocessing.get_context("spawn").Pool(min(16, os.cpu_count())) as pool:
                res = pool.map(_verdict, todo, chunksize=1)
        else:
            res = [_verdict(b) for b in todo]
        for b, v in zip(todo, res):
            _VERDICTS[_key(b)] = v
    return [_VERDICTS[_key(b)] for b in bodies]


# ================================================================ tests
def _digest(bodies):
    h = hashlib.sha256()
    for b in bodies:
        h.update(len(b).to_bytes(8, "little") + b)
    return h.hexdigest()


def test_large_corpus_shape():
    bodies = large_corpus()
    sizes = [len(b) for b in bodies]
    assert len(bodies) >= 300 and min(sizes) > 65536 and max(sizes) <= 8 * MIB
    assert 45 * MIB <= sum(sizes) <= 80 * MIB, sum(sizes)
    assert large_corpus.__wrapped__(6) == bodies[:6] and large_corpus.__wrapped__(6, seed=42) != bodies[:6]   # deterministic by seed
    joined = b"".join(bodies[:60])
    for needle in (b"\\n", b'\\"', b"\\\\", b"\\u", b'"rank_fields"', b'"metadata"', "東京".encode(), "𝔘".encode(), b'\n  "'):
        assert needle in joined, needle
    for b in bodies[:40] + bodies[4:6]:   # json.loads agrees with the oracle: every one decodes
        d = json.loads(b)
        assert 50 <= len(d["documents"]) <= 5000 and all(200 <= len(x) <= 4000 for x in d["documents"])
    assert [v for v, _ in verdicts(bodies[5:25])] == [Q.OK] * 20


def test_near_limit_bodies():
    bl = near_limit_bodies()
    assert [len(b) for b, _ in bl] == [LIMIT - 1, LIMIT - 100, LIMIT - 8193, LIMIT]
    assert sized_body(100000, seed=3) == sized_body(100000, seed=3)
    json.loads(sized_body(100000, seed=3))


def test_boundary_corpus():
    corpus = boundary_corpus()
    assert _digest(b for _, b in corpus) == _digest(b for _, b in boundary_corpus())
    assert all(len(b) % TILE in (1, TILE - 1) for _, b in corpus)
    labels = [l for l, _ in corpus]
    assert {int(l.split()[0][3:]) for l in labels if l.startswith("run")} == set(range(1, 71))
    # the feature's first byte is on the boundary at offset 0
    for l, b in corpus:
        if l.startswith("u_escape thread@+0"):
            assert b[3200:3202] == b"\\u"
        if l.startswith("run33 tile@+0"):
            assert b[8192 - 33:8193] == b"\\" * 33 + b'"'
    # the oracle against json.loads on a sample: where json.loads decodes, the oracle's verdict is OK, except for a number in
    # documents (the decoder's type error); where it does not, FAIL (no control bytes, depth 2)
    sample = corpus[::7]
    for (l, b), (v, _) in zip(sample, verdicts([b for _, b in sample])):
        try:
            json.loads(b)
            ok = not l.startswith("number_elem")
        except ValueError:
            ok = False
        assert v == (Q.OK if ok else Q.FAIL), (l, v)


def test_splice_corpus():
    bodies = splice_corpus()
    assert len(bodies[0]) > 3 * MIB and bodies[0].endswith(b'"model":"rerank-v3.5"}')
    vs = [v for v, _ in verdicts(bodies)]
    assert vs[:9] == [Q.OK] * 9 and vs[9] == Q.OUT and vs[10] == Q.OUT and vs[11] == Q.OK
    for b, v in zip(bodies, vs):
        if v == Q.OK:
            json.loads(b)
