"""Malformed requests for the one-CTA-per-request scans of aigw_{chat,embeddings,rerank}_translate_large_*, with each defect at a
thread, warp or tile boundary of the scan (test_large_scan_defects_gpu.py feeds them through the GPU), and their self-checks.

The scans stream a body in 8 KiB tiles, 32 bytes per thread, and carry the parity of a backslash run and the in-string state
across thread, warp and tile boundaries.  A carry that is wrong at a boundary still lets most bodies through; what shows it is a
defect next to the boundary.  So:

  probes        a short structure-dense fragment (numbers, true / false / null, empty and nested containers, a key, a string with
                \\" \\\\ and a non-ASCII letter) where each kernel really looks, padded in front with white space so that each of its
                bytes in turn lies on a boundary: thread 3200 (not a warp), warp 5120 (not a tile), tiles 8192 and 16384, and 73728,
                one tile past the translate pass's 64 KiB ceiling.  The byte on the boundary is deleted, duplicated or replaced.
  truncations   a realistic body of about 80 KB cut within +-40 bytes of each boundary and at k * 8192 +- 1, also with a lone
                trailing backslash and with trailing white space
  runs          31 ... 16385 backslashes and a quote inside a string, starting on or ending at a thread, warp or tile boundary.
                Each run has a valid twin and a malformed twin: reading the run's parity wrongly turns the valid twin into a
                syntax error and the malformed twin into a valid body.
  near 16 MiB   bodies of 16 MiB - 1 with the probe (intact, or with a defect) in the last tile

`scan_model` restates the scan's per-byte escape and in-string state (count_tokens in test_translate_edges_cpu.py, as token
lists) with switches that drop one carry at one kind of boundary; the corpus must tokenise differently under every switch."""
import functools
import hashlib
import json

import numpy as np
import pytest

import _oracle as O
import test_chat_large_cpu as CL
import test_embeddings_large_cpu as EL
import test_rerank_large_cpu as RL
import test_translate_edges_cpu as E

MIB = 1 << 20
THREAD, WARP, TILE = 32, 1024, 8192
# (kind, byte offset): 3200 starts a thread but not a warp, 5120 a warp but not a tile; 73728 is the first tile boundary past
# the translate pass's 64 KiB ceiling
BOUNDS = (("thread", 3200), ("warp", 5120), ("tile", 8192), ("tile2", 16384), ("ceiling", 73728))
KERNELS = ("chat", "emb", "rerank")

# ================================================================ probes and where they go
# a member value: numbers, literals, empty and nested containers, a key, a string holding \" \\ and é
PROBE = b'{"k":[-0,-2.5e-3,10,true,false,null,{},[],[[1],{"a":[null]}]],"s":"q\\"r\\\\s\xc3\xa9"}'
# the same for tool parameters, whose numbers the translate pass re-prints: -2.5e-3 spelled as strconv prints it
PARAM_PROBE = b'{"k":[-0,-0.0025,10,true,false,null,{},[],[[1],{"a":[null]}]],"s":"q\\"r\\\\s\xc3\xa9"}'
# elements of a flat []string (nulls allowed): the parallel neighbour rule of the input / documents arrays
STR_PROBE = b'"a",null,"q\\"r\\\\s\xc3\xa9","",null,"-2.5e-3","{}[]:,","tru e",null'
# members around top_n
TOPN_PROBE = b'"x_a":{"k":[-0,-2.5e-3,true,false,null,{},[]]},"top_n":10,"x_b":[[1],{"a":[null]}],"x_s":"q\\"r\\\\s\xc3\xa9"'


@functools.lru_cache(maxsize=None)
def _chat_rest():
    """the members of a realistic agent transcript, without a model, to follow an unknown member"""
    return CL.long_chat(21, 4000, "true", model=False)[1:]


def _sites():
    """kernel -> {site: (head, pre, probe, post)}: the body is head + white space + pre + probe + post"""
    return {
        "chat": {
            "unknown": (b'{"model":"gpt-4o-mini",', b'"x_probe":', PROBE, b"," + _chat_rest()),
            "part": (b'{"model":"gpt-4o-mini","messages":[{"role":"system","content":"be brief"},{"role":"user","content":[{"type":"text","text":"hi"},',
                     b'{"type":"text","text":"a\\"b","x_probe":', PROBE,
                     b'},{"type":"text","text":"tail","cache_control":{"type":"ephemeral"}}]}],"stream":true,"temperature":0.5}'),
            "params": (b'{"model":"gpt-4o-mini","messages":[{"role":"user","content":"hi"}],"tools":[{"type":"function","function":{"name":"f","description":"d",',
                       b'"parameters":', PARAM_PROBE, b'}}],"tool_choice":"auto","max_tokens":64}'),
        },
        "emb": {
            "input": (b'{"model":"text-embedding-3-small","input":[', b"", STR_PROBE, b',"tail"],"dimensions":256}'),
            "item": (b'{"model":"text-embedding-004","input":[{"content":"a"},', b'{"content":"b","task_type":"RETRIEVAL_DOCUMENT","title":"t","x_probe":',
                     PROBE, b"}]}"),
            "unknown": (b'{"model":"text-embedding-3-small",', b'"x_probe":', PROBE, b',"input":["a","b\\u00e9"],"encoding_format":"float"}'),
        },
        "rerank": {
            "documents": (b'{"model":"rerank-v3.5","query":"refund policy","documents":[', b"", STR_PROBE, b',"tail"],"top_n":2}'),
            "top_n": (b'{"model":"rerank-v3.5","query":"q","documents":["a","b"],', b"", TOPN_PROBE, b"}"),
            "unknown": (b'{"model":"rerank-v3.5",', b'"x_probe":', PROBE, b',"query":"q","documents":["a","b"]}'),
        },
    }


def _pad(n):
    """n bytes of JSON white space (a newline every 80 bytes): no token, no escape, no string"""
    return ((b" " * 79 + b"\n") * (n // 80 + 1))[:n]


def probe_body(kernel, site, bound, k):
    """the valid body whose probe byte k lies on byte `bound`"""
    head, pre, probe, post = _sites()[kernel][site]
    n = bound - k - len(head) - len(pre)
    assert n >= 0, (kernel, site, bound, k)
    body = head + _pad(n) + pre + probe + post
    assert body[bound] == probe[k]
    return body


# the bytes a probe byte is replaced with: mutants()'s structural set, a control byte, a raw newline, an invalid UTF-8 byte and
# bytes that continue numbers, literals and \u escapes
MUT_BYTES = E.MUTATION_BYTES + b"\x01\n\xffe-.0u"


def _mutations(body, at):
    """(name, body): the byte at `at` deleted, duplicated or replaced (identical results dropped)"""
    out = [("del", body[:at] + body[at + 1:]), ("dup", body[:at + 1] + body[at:])]
    out += [("rep%02x" % c, body[:at] + bytes([c]) + body[at + 1:]) for c in MUT_BYTES if c != body[at]]
    return out


@functools.lru_cache(maxsize=None)
def probe_corpus(kernel):
    """(label, bound, at, body) for every site, boundary, probe byte on it and mutation; label = 'site kind k mutation'"""
    out, seen = [], set()
    for site, (_, _, probe, _) in _sites()[kernel].items():
        for kind, bound in BOUNDS:
            for k in range(len(probe)):
                for name, m in _mutations(probe_body(kernel, site, bound, k), bound):
                    if m not in seen:
                        seen.add(m)
                        out.append(("%s %s %d %s" % (site, kind, k, name), bound, bound, m))
    return tuple(out)


# ================================================================ truncations
@functools.lru_cache(maxsize=None)
def truncation_base(kernel):
    """a realistic valid body of 80-100 KB"""
    if kernel == "chat":
        return CL.long_chat(33, 80000, "true")
    if kernel == "emb":
        import random
        r = random.Random(3)
        return json.dumps({"model": "text-embedding-3-small", "input": [EL._text(r, 50, 900) for _ in range(160)], "dimensions": 256},
                          ensure_ascii=True).encode()
    return RL.large_request(17, 85000)


def truncation_cuts(n):
    cuts = {b + d for _, b in BOUNDS for d in range(-40, 41)} | {k * TILE + d for k in range(1, n // TILE + 1) for d in (-1, 1)}
    return sorted(c for c in cuts if 0 < c < n)


@functools.lru_cache(maxsize=None)
def truncation_corpus(kernel):
    """(label, bound, at, body): the base cut at each length, then with a trailing backslash, then with trailing white space"""
    base = truncation_base(kernel)
    out = []
    for c in truncation_cuts(len(base)):
        for tag, tail in (("cut", b""), ("bs", b"\\"), ("ws", b" \n\t ")):
            out.append(("%s %d" % (tag, c), c, c, base[:c] + tail))
    return tuple(out)


# ================================================================ long backslash runs
RUN_LENGTHS = (31, 32, 33, 1023, 1024, 1025, 8191, 8192, 8193, 16385)


def _run_site(kernel):
    """(head, rest): the run sits in a string that head opens; rest follows the string when it closes"""
    return {"chat": (b'{"model":"gpt-4o-mini","messages":[{"role":"user","content":"', b'}],"stream":true}'),
            "emb": (b'{"model":"text-embedding-3-small","input":["', b',"z"]}'),
            "rerank": (b'{"model":"rerank-v3.5","query":"q","documents":["', b',"z"]}')}[kernel]


def _end_bound(kind, n):
    """the first boundary of this kind with room for a run of n bytes (and the head) before it"""
    w = n + 96
    if kind == "thread":
        return (w + WARP - 1) // WARP * WARP + 96
    if kind == "warp":
        return (w + TILE - 1) // TILE * TILE + WARP
    return (w + TILE - 1) // TILE * TILE


def run_body(kernel, n, kind, where, twin):
    """a string holding n backslashes and a quote, the run starting on (where='start') or ending at (where='end') a boundary of
    this kind.  An even run leaves the quote closing the string, an odd one escapes it.  The valid twin follows the quote with
    what makes the body valid under the run's true parity, the malformed twin with what makes it valid under the other parity."""
    head, rest = _run_site(kernel)
    b = dict(BOUNDS[:3])[kind] if where == "start" else _end_bound(kind, n)
    start = b if where == "start" else b - n
    closes = n % 2 == 0
    cont = b'a"' if closes != (twin == "valid") else b""
    body = head + b"a" * (start - len(head)) + b"\\" * n + b'"' + cont + rest
    assert body[start:start + n] == b"\\" * n and body[start - 1] != 0x5C and body[start + n] == 0x22
    return body, b, start


@functools.lru_cache(maxsize=None)
def run_corpus(kernel):
    """(label, bound, start of the run, body)"""
    out = []
    for n in RUN_LENGTHS:
        for kind in ("thread", "warp", "tile"):
            for where in ("start", "end"):
                for twin in ("valid", "malformed"):
                    body, b, start = run_body(kernel, n, kind, where, twin)
                    out.append(("run%d %s %s %s" % (n, kind, where, twin), b, start, body))
    return tuple(out)


# ================================================================ near 16 MiB
@functools.lru_cache(maxsize=None)
def near_limit_corpus(kernel):
    """(label, bound, at, body): 16 MiB - 1 bytes, a long string member first, the probe in the last tile: intact, and with a
    syntax error in its structure, far from its escapes: the ']' of its '[[1]' deleted, the ':' after its key "k" made a ',',
    the quote that opens "k" duplicated"""
    head = {"chat": b'{"model":"gpt-4o-mini","messages":[{"role":"user","content":"hi"}],"x_pad":"',
            "emb": b'{"model":"text-embedding-3-small","input":["a"],"x_pad":"',
            "rerank": b'{"model":"rerank-v3.5","query":"q","documents":["a"],"x_pad":"'}[kernel]
    tail = b'","x_probe":' + PROBE + b"}"
    i_br, i_colon, i_q = tail.index(b"[[1]") + 3, tail.index(b'"k":') + 3, tail.index(b'"k":')
    tails = (("near intact", tail, None), ("near del]", tail[:i_br] + tail[i_br + 1:], i_br), ("near :->,", tail[:i_colon] + b"," + tail[i_colon + 1:], i_colon),
             ("near dup\"", tail[:i_q] + b'"' + tail[i_q:], i_q))
    pad = bytes(b"abcdefgh "[i % 9] for i in range(16 * MIB))
    out = []
    for name, t, i in tails:
        n = (16 * MIB - 1) - len(head) - len(t)
        body = head + pad[:n] + t
        p0 = len(body) - len(t)
        out.append((name, p0, p0 + (i or 0), body))
    return tuple(out)


def defect_corpus(kernel, near=False):
    """every generated body of a kernel: probes, truncations, runs (and the 16 MiB ones)"""
    return probe_corpus(kernel) + truncation_corpus(kernel) + run_corpus(kernel) + (near_limit_corpus(kernel) if near else ())


def _escaped_or_backslash(body, at):
    """byte `at` is a backslash, or an odd run of backslashes precedes it"""
    if body[at] == 0x5C:
        return True
    run = 0
    while at - run - 1 >= 0 and body[at - run - 1] == 0x5C:
        run += 1
    return run % 2 == 1


def defect_touches_escape(kernel, label, at):
    """the defect changes which bytes are backslashes or escaped: it writes a backslash, or it deletes, duplicates or replaces
    a backslash or an escaped byte, or a cut leaves a backslash last.  Only such a defect may turn a syntax error into an
    escape decline; the backslash runs are made to be read (their defect is the parity) and count as not touching."""
    if label.startswith("run"):
        return False
    if label.startswith("near"):
        return _escaped_or_backslash(near_limit_corpus(kernel)[0][3], at)
    if label.split()[0] in ("cut", "bs", "ws"):
        tag, c = label.split()
        return tag == "bs" or truncation_base(kernel)[int(c) - 1] == 0x5C
    site, kind, k, name = label.split()
    orig = probe_body(kernel, site, dict(BOUNDS)[kind], int(k))
    return name == "rep5c" or _escaped_or_backslash(orig, at)


# ================================================================ the scan model
OPEN, CLOSE, SCALAR = 1, 2, 3
_OPS = np.zeros(256, bool); _OPS[list(b"{}[]:,")] = True
_WS = np.zeros(256, bool); _WS[list(b" \t\n\r")] = True
_ESC_OK = np.zeros(256, bool); _ESC_OK[list(b'"\\/bfnrtu')] = True
_HEX = np.zeros(256, bool); _HEX[list(b"0123456789abcdefABCDEF")] = True
# the carries a switch drops: (state, boundary kind); 'allbs' drops the escape carry through a thread that is all backslashes
SWITCHES = tuple((s, k) for s in ("escape", "string") for k in ("thread", "warp", "tile")) + ("allbs",)


def scan_model(body, lo=0, hi=None, in_str=False, drop=()):
    """The scan's state over body[lo:hi] (absolute offsets; lo must be a point where no backslash run is open, and `in_str` the
    string state there).  A byte is escaped when an odd run of backslashes precedes it, inside strings or not; an unescaped quote
    toggles the string; tokens are the unescaped quotes, structural bytes outside strings and the first byte of every run of
    scalar bytes outside strings, as count_tokens counts them.  `drop` holds switches from SWITCHES: the escape carry or the
    in-string state is lost at every boundary of that kind (thread: a thread start that is no warp start; warp: a warp start
    that is no tile start; tile: a tile start), as a scan that forgot that carry would compute it.
    Returns (a, esc, inside, positions of the tokens, their types)."""
    hi = len(body) if hi is None else hi
    n = hi - lo
    a = np.frombuffer(body, np.uint8, n, lo)
    pos = np.arange(lo, hi)
    idx = np.arange(n)
    bs = a == 0x5C
    reset_e = np.zeros(n, bool)
    reset_s = np.zeros(n, bool)
    if drop:
        tile = pos % TILE == 0
        warp = (pos % WARP == 0) & ~tile
        thread = (pos % THREAD == 0) & (pos % WARP != 0)
        kinds = {"thread": thread, "warp": warp, "tile": tile}
        for d in drop:
            if d == "allbs":
                cs = np.concatenate(([0], np.cumsum(bs)))
                full = np.zeros(n, bool)
                ok = (pos % THREAD == 0) & (idx >= THREAD)
                full[ok] = cs[idx[ok]] - cs[idx[ok] - THREAD] == THREAD
                reset_e |= full
            elif d[0] == "escape":
                reset_e |= kinds[d[1]]
            else:
                reset_s |= kinds[d[1]]
    last_nb = np.maximum.accumulate(np.where(~bs, idx, -1))
    prev_nb = np.concatenate(([-1], last_nb[:-1]))
    last_r = np.maximum.accumulate(np.where(reset_e, idx, 0))
    esc = ((idx - np.maximum(prev_nb + 1, last_r)) & 1).astype(bool)   # the run of backslashes before the byte is odd
    uq = (a == 0x22) & ~esc
    cq = np.cumsum(uq)
    if reset_s.any():
        last_s = np.maximum.accumulate(np.where(reset_s, idx, -1))
        before = np.where(last_s > 0, cq[np.maximum(last_s, 1) - 1], 0)
        ps = ((cq - before) & 1).astype(bool) ^ (bool(in_str) & (last_s < 0))
    else:
        ps = (cq & 1).astype(bool) ^ bool(in_str)
    inside, out = ps & ~uq, ~ps & ~uq
    op, ws = _OPS[a], _WS[a]
    sc = out & ~op & ~ws
    tok = (op & out) | uq | (sc & ~np.concatenate(([False], sc[:-1])))
    ty = np.where(uq, np.where(ps, OPEN, CLOSE), np.where(op, a, SCALAR))
    return a, esc, inside, pos[tok], ty[tok]


def scan_flags(body):
    """what the scan itself declines for, by the model: a control byte inside a string, an invalid escape inside a string, a key
    (a string followed by ':') holding an escaped byte"""
    a, esc, inside, tp, tt = scan_model(body)
    flags = set()
    if (inside & (a < 0x20)).any():
        flags.add("ctrl")
    e = np.flatnonzero(esc & inside)
    bad = ~_ESC_OK[a[e]]
    for i in e[(a[e] == ord("u")) & ~bad]:
        bad_u = i + 4 >= len(a) or not _HEX[a[i + 1:i + 5]].all()
        if bad_u:
            flags.add("escape")
            break
    if bad.any():
        flags.add("escape")
    if len(tt) > 2:
        ce = np.concatenate(([0], np.cumsum(esc & inside)))
        k = np.flatnonzero((tt[:-2] == OPEN) & (tt[1:-1] == CLOSE) & (tt[2:] == ord(":")))
        if (ce[tp[k + 1]] != ce[tp[k]]).any():
            flags.add("escaped_key")
    return flags


def model_window(kernel, label, bound, at, body):
    """(lo, hi, in_str) around a defect: from inside the white space in front of the probe, or from the string text in front
    of the run, to past it"""
    if label.startswith("run"):
        return at - 48, min(len(body), bound + 64 if at < bound else at + int(label.split()[0][3:]) + 64), True
    site, _, k, _ = label.split()
    head, pre, _, _ = _sites()[kernel][site]
    lo = bound - int(k) - len(pre) - 32
    assert lo >= len(head) and not body[lo:bound - int(k) - len(pre)].strip()
    return lo, min(len(body), bound + 128), False


def carry_reached(kernel, label, bound, at, body, sw):
    """near its boundary, the body tokenises differently, or has other escaped bytes inside strings (the bytes the scan
    validates as escapes), when the scan drops this carry"""
    lo, hi, ins = model_window(kernel, label, bound, at, body)
    _, e0, i0, p0, t0 = scan_model(body, lo, hi, ins)
    _, e1, i1, p1, t1 = scan_model(body, lo, hi, ins, (sw,))
    return not (np.array_equal(p0, p1) and np.array_equal(t0, t1) and np.array_equal(e0 & i0, e1 & i1))


def digest(items):
    h = hashlib.sha256()
    for it in items:
        b = it[-1]
        h.update(it[0].encode() + len(b).to_bytes(8, "little") + b)
    return h.hexdigest()


# ================================================================ oracle verdicts
def oracle_status(kernel, body):
    """OK / 400 / other, in the oracle's terms for the kernel's OpenAI-shaped configuration"""
    if kernel == "chat":
        s = O.chat_translate("openai", body).status
    elif kernel == "emb":
        s = O.embeddings_translate("openai", body).status
    else:
        v = RL.verdicts([body])[0][0]
        import _rerank_oracle as Q
        s = O.OK if v == Q.OK else O.MALFORMED_400 if v == Q.FAIL else O.DECLINED
    return "ok" if s == O.OK else "400" if s == O.MALFORMED_400 else "other"


# ================================================================ self-checks
# pinned: a change to a generator changes what the GPU test compares, and shows here
DIGESTS = {
    "chat": "e8f8038f0ac81b29e738e50a44af67cfee0d0726372963671fb6e0519c5854f6",
    "emb": "657f27b74046ccee2b0785657c73f2095349dcb4bdf0151c6039967d84f8862a",
    "rerank": "107a6958ba1eef0b849f3bf5274484cd4e07c12148a792e0d04b9c5d7a525e97",
}


@pytest.mark.parametrize("kernel", KERNELS)
def test_generators_are_deterministic(kernel):
    d = digest(defect_corpus(kernel))
    assert d == DIGESTS[kernel], (kernel, d)


@pytest.mark.parametrize("kernel", KERNELS)
def test_probes_sit_on_their_boundaries(kernel):
    for site, (_, _, probe, _) in _sites()[kernel].items():
        for _, bound in BOUNDS:
            for k in range(len(probe)):
                b = probe_body(kernel, site, bound, k)
                assert b[bound - k:bound - k + len(probe)] == probe
                json.loads(b)
    corpus = probe_corpus(kernel)
    for label, bound, at, m in corpus[::97]:
        site, kind, k, name = label.split()
        assert dict(BOUNDS)[kind] == bound == at
        probe = _sites()[kernel][site][2]
        orig = probe_body(kernel, site, bound, int(k))
        assert orig[bound] == probe[int(k)]
        if name == "del":
            assert m == orig[:at] + orig[at + 1:]
        elif name == "dup":
            assert m[at] == m[at + 1] == orig[at] and len(m) == len(orig) + 1
        else:
            assert m[at] == int(name[3:], 16) and len(m) == len(orig) and m[:at] == orig[:at] and m[at + 1:] == orig[at + 1:]
    # every site, kind and probe byte is there, each with the 19 mutations less the identical ones
    n = sum(len(p) * len(BOUNDS) for _, _, p, _ in _sites()[kernel].values())
    assert n * 15 < len(corpus) <= n * 19
    sizes = {kind: [len(b) for l, _, _, b in corpus if l.split()[1] == kind] for kind, _ in BOUNDS}
    assert max(sizes["thread"]) <= 65536 < min(sizes["ceiling"])


@pytest.mark.parametrize("kernel", KERNELS)
def test_truncations_runs_and_limit_shapes(kernel):
    base = truncation_base(kernel)
    json.loads(base)
    assert 78000 < len(base) < 110000
    tc = truncation_corpus(kernel)
    assert {c for _, _, c, _ in tc} == set(truncation_cuts(len(base)))
    for l, _, c, b in tc:
        assert b.startswith(base[:c]) and b[c:] in (b"", b"\\", b" \n\t ")
    rc = run_corpus(kernel)
    assert len(rc) == len(RUN_LENGTHS) * 3 * 2 * 2
    for l, bound, start, b in rc:
        n, kind, where, twin = l[3:].split()
        n = int(n)
        assert b[start:start + n] == b"\\" * n and b[start + n] == 0x22
        assert (start if where == "start" else start + n) == bound
        assert bound % {"thread": THREAD, "warp": WARP, "tile": TILE}[kind] == 0
        assert kind == "tile" or bound % {"thread": WARP, "warp": TILE}[kind] != 0
        try:
            json.loads(b)
            ok = True
        except ValueError:
            ok = False
        assert ok == (twin == "valid"), l
    for l, p0, at, b in near_limit_corpus(kernel):
        assert len(b) == 16 * MIB - 1 and at >= len(b) - TILE and p0 >= len(b) - TILE
    assert json.loads(near_limit_corpus(kernel)[0][3])["x_probe"]["s"] == 'q"r\\sé'


@pytest.mark.parametrize("kernel", KERNELS)
def test_few_defects_touch_an_escape(kernel):
    """only defects that write, remove or shift a backslash or an escaped byte are excused from a 400: a backslash written in
    place of any probe byte, and the probe's five escape bytes (one in ten probe bodies); a lone trailing backslash and a cut
    right after a backslash; none of the 16 MiB - 1 defects, which sit on structure with no escape nearby"""
    pc = probe_corpus(kernel)
    touched = [l for l, _, at, _ in pc if defect_touches_escape(kernel, l, at)]
    assert 0.08 * len(pc) < len(touched) < 0.12 * len(pc), (len(touched), len(pc))
    assert all(l.endswith("rep5c") or int(l.split()[2]) in _escape_bytes(_sites()[kernel][l.split()[0]][2]) for l in touched)
    tc = truncation_corpus(kernel)
    assert sum(defect_touches_escape(kernel, l, at) for l, _, at, _ in tc) - sum(l.startswith("bs") for l, *_ in tc) < 0.05 * len(tc)
    near = near_limit_corpus(kernel)
    assert not any(defect_touches_escape(kernel, l, at) for l, _, at, _ in near)
    for l, _, at, b in near[1:]:
        assert b"\\" not in b[at - 8:at + 9] and not scan_flags(b), l
        assert not _json_valid(b)


def _escape_bytes(probe):
    return {i for i in range(len(probe)) if _escaped_or_backslash(probe, i)}


def _json_valid(b):
    try:
        json.loads(b)
        return True
    except ValueError:
        return False


def test_scan_model_counts_tokens_as_the_index_stage():
    """the model's token count is count_tokens' on the corpus and on known answers, and a window of a body tokenises as the
    whole body does inside it"""
    for kernel in KERNELS:
        for l, bound, at, b in defect_corpus(kernel)[::211]:
            assert len(scan_model(b)[3]) == E.count_tokens(b), (kernel, l)
    cases = [(b'{"a\\"b":"c\\\\"}', 7), (b'"a\\\\\\"b"', 2), (b'\\"x', 1), (b'{"k":-1.5e3,"v":[null]}', 13)]
    for b, want in cases:
        assert len(scan_model(b)[3]) == want
    # a window gives the tokens of the whole body inside it
    b = probe_corpus("chat")[500][3]
    _, _, _, p, t = scan_model(b)
    _, _, _, pw, tw = scan_model(b, 3000, 3400)
    sel = (p >= 3000) & (p < 3400)
    assert np.array_equal(p[sel], pw) and np.array_equal(t[sel], tw)


def test_scan_model_switches():
    """each switch changes exactly the carry it names"""
    run = b'"' + b"a" * 30 + b"\\" + b'"' + b"a" * 40 + b'"'   # the escaped quote is byte 32: a thread boundary
    assert not np.array_equal(scan_model(run)[3], scan_model(run, drop=(("escape", "thread"),))[3])
    assert np.array_equal(scan_model(run)[3], scan_model(run, drop=(("escape", "warp"),))[3])
    s = b" " * 8100 + b'"' + b"a" * 200 + b'",1'   # a string open across the tile boundary, and across no other warp start
    assert not np.array_equal(scan_model(s)[3], scan_model(s, drop=(("string", "tile"),))[3])
    assert np.array_equal(scan_model(s)[3], scan_model(s, drop=(("string", "warp"),))[3])
    w = b'"' + b"a" * (WARP - 2) + b"\\" + b'"' + b'"'   # the escaped quote is byte 1024: a warp boundary
    assert not np.array_equal(scan_model(w)[3], scan_model(w, drop=(("escape", "warp"),))[3])
    assert np.array_equal(scan_model(w)[3], scan_model(w, drop=(("escape", "thread"),))[3])
    # 33 backslashes ending at 64: the thread 32-63 is all backslashes, the quote at 64 is escaped
    r = b'"' + b"a" * 30 + b"\\" * 33 + b'"a"'
    assert not np.array_equal(scan_model(r)[3], scan_model(r, drop=("allbs",))[3])


# the share of OK and of 400 among the probe bodies per boundary kind, floors a little below what the oracle gives every 7th
# one: chat 12-13 % OK / 87-88 % 400, embeddings 18-19 % / 81-82 %, rerank 18-20 % / 78-79 % (2-3 % outside the decoder's subset)
VERDICT_FLOORS = {
    "chat": (0.10, 0.80),
    "emb": (0.15, 0.75),
    "rerank": (0.15, 0.70),
}


@pytest.mark.parametrize("kernel", KERNELS)
def test_both_verdicts_are_well_represented(kernel):
    """every seventh probe body's oracle verdict: both OK and 400 are common at every boundary kind"""
    corpus = probe_corpus(kernel)[::7]
    if kernel == "rerank":
        RL.verdicts([b for *_, b in corpus])
    split = {}
    for l, _, _, b in corpus:
        s = split.setdefault(l.split()[1], {"ok": 0, "400": 0, "other": 0})
        s[oracle_status(kernel, b)] += 1
    print("\n%s: oracle verdicts of every 7th probe body by boundary kind %s" % (kernel, split))
    lo_ok, lo_400 = VERDICT_FLOORS[kernel]
    for kind, s in split.items():
        n = sum(s.values())
        assert s["ok"] >= lo_ok * n and s["400"] >= lo_400 * n, (kernel, kind, s)
    # the valid twins of the runs are OK, the malformed twins 400
    rc = run_corpus(kernel)
    if kernel == "rerank":
        RL.verdicts([b for *_, b in rc])
    for l, _, _, b in rc:
        assert oracle_status(kernel, b) == ("ok" if l.endswith(" valid") else "400"), l


@pytest.mark.parametrize("kernel", KERNELS)
def test_corpus_reaches_every_carry(kernel):
    """for every switch and every boundary kind it drops a carry at, many bodies tokenise differently near their boundary
    under the switch than under the correct model"""
    corpus = probe_corpus(kernel) + run_corpus(kernel)
    reached = {}
    for l, bound, at, b in corpus:
        kind = l.split()[1]
        bk = "tile" if kind in ("tile", "tile2", "ceiling") else kind
        for sw in SWITCHES:
            if sw == "allbs":
                if not l.startswith("run") or int(l.split()[0][3:]) < 33:
                    continue
            elif sw[1] != bk:
                continue
            key = (sw if sw == "allbs" else "%s@%s" % sw, kind)
            reached.setdefault(key, [0, 0])[1] += 1
            if carry_reached(kernel, l, bound, at, b, sw):
                reached[key][0] += 1
    print("\n%s: bodies that tokenise differently when a carry is dropped (switch, kind): [differ, bodies] %s" % (kernel, reached))
    for kind, _ in BOUNDS:
        bk = "tile" if kind in ("tile2", "ceiling") else kind
        for st in ("escape", "string"):
            hit, n = reached[("%s@%s" % (st, bk), kind)]
            assert hit >= 50, (kernel, st, kind, hit, n)
    for kind in ("thread", "warp", "tile"):
        assert reached[("allbs", kind)][0] >= 4, (kernel, kind, reached[("allbs", kind)])
