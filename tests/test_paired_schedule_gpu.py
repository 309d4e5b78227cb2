"""The paired translate schedule of a device call of several sub-batches (the index of sub-batch k+1 and the emit of sub-batch k in one
launch, chat_kernel.cu launch_cls) against the serial schedule the stage profile runs (aigw_chat_set_profile), per document: status,
reason, record bytes, model span, flags and body kind.  out_off is not compared: the bump allocator places records in completion order.
Each case crosses several sub-batch boundaries; a sample, including the documents on either side of every boundary, is checked
against the oracle."""
import numpy as np
import pytest

import _oracle as O
import _workload as W
from test_bench_paths_gpu import OK, DeviceCorpus, check_layout, records

pytestmark = pytest.mark.gpu
PAIR_SUB = 229376   # documents per sub-batch of the paired schedule when the workspace cap does not bound it (chat_kernel.cu kPairSubDocs);
                    # a call pairs from two such sub-batches on


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def both_schedules(ctx, cfg, arena, offs, lens, max_len=None, doc_map=None):
    """(records, results, launches) of the call as it runs by default, then of the same call with the stage profile on"""
    n = len(lens)
    max_len = max_len or int(lens.max())
    dc = DeviceCorpus(ctx, arena, offs, lens)
    try:
        d_map = None
        if doc_map is not None:
            d_map = dc._alloc(doc_map.nbytes); ctx.h2d(d_map, doc_map)

        def call():
            dc.reset()
            if d_map is None:
                ctx.chat_translate_device(cfg, dc.d_in, dc.d_off, dc.d_len, n, max_len, dc.d_out, dc.out_cap, dc.d_res, dc.d_used)
            else:
                ctx.chat_translate_device_mapped(cfg, dc.d_in, dc.d_off, dc.d_len, d_map, 0, n, max_len, dc.d_out, dc.out_cap, dc.d_res, dc.d_used)
            launches = ctx.chat_last_profile()["launches"]
            res, out = dc.fetch()
            return records(res, out), res, launches

        paired = call()
        ctx.chat_set_profile(True)
        try:
            serial = call()
        finally:
            ctx.chat_set_profile(False)
    finally:
        dc.free()
    return paired, serial


def check_paired(paired, serial, n):
    recs, res, launches = paired
    srecs, _, slaunches = serial
    # I(0), then sort + walk + (paired launch or the last emit) per sub-batch; the serial schedule: 4 launches per sub-batch
    assert launches % 3 == 1 and launches >= 7, launches
    assert slaunches % 4 == 0, slaunches
    assert (res["status"] != 255).all(), "a document the paired call never reached"
    check_layout(res)
    assert len(recs) == n
    bad = [i for i in range(n) if recs[i] != srecs[i]]
    assert not bad, (len(bad), bad[:10])
    return (launches - 1) // 3


def oracle_sample(schema, arena, offs, lens, recs, idx, model_override=""):
    for i in idx:
        b = bytes(arena[int(offs[i]):int(offs[i]) + int(lens[i])])
        st, _, rec, *_ = recs[i]
        if st != OK:   # declined bodies go to the reference's own translator; 400 / 422 statuses are compared with the serial schedule
            continue
        t = O.chat_translate(schema, b, model_override=model_override)
        assert t.status == O.OK, (i, t.err)
        pl = len(t.path.encode())
        assert rec[:pl].decode() == t.path and rec[pl:] == (t.body if t.body_kind == O.BYTES else b""), i


def boundaries(nsb, n, step=997):
    """documents on either side of each sub-batch boundary (the call cuts nsb equal sub-batches) and every step-th one"""
    sub = -(-n // nsb)
    near = set()
    for k in range(1, nsb):
        near |= set(range(max(0, k * sub - 8), min(n, k * sub + 8)))
    return sorted(near | set(range(0, n, step)))


def test_bench_shape(ctx):
    """the headline call's shape: 4 KB Bedrock bodies (5120 class, seed 2) over three sub-batches"""
    n = 2 * PAIR_SUB + 1000
    arena, offs, lens = W.chat_corpus(2, 0, n)
    assert 2048 < int(lens.max()) <= 5120
    paired, serial = both_schedules(ctx, ctx.cfg("aws-bedrock"), arena, offs, lens)
    assert check_paired(paired, serial, n) == 3
    assert (paired[1]["status"] == OK).all()
    oracle_sample("aws-bedrock", arena, offs, lens, paired[0], boundaries(3, n))


@pytest.mark.parametrize("tail", [5, 1])
def test_2048_class_uneven_split(ctx, tail):
    """a call just past two full sub-batches: it is cut into three equal ones (not two full ones and a few documents), whose
    sizes differ by one when the count does not divide"""
    n = 2 * PAIR_SUB + tail
    arena, offs, lens = W.chat_corpus(13, 0, n, target=1024)
    assert int(lens.max()) <= 2048
    paired, serial = both_schedules(ctx, ctx.cfg("aws-bedrock"), arena, offs, lens, max_len=2048)
    nsb = check_paired(paired, serial, n)
    assert nsb == -(-n // PAIR_SUB)
    oracle_sample("aws-bedrock", arena, offs, lens, paired[0], boundaries(nsb, n) + [n - 1])


@pytest.mark.parametrize("cls", [17408, 65536])
def test_large_classes_under_workspace_cap(ctx, cls):
    """the class is the call's max_len: small bodies, a workspace bounded by the 3 GiB cap.  At 17408 two slots of the cap hold
    fewer than PAIR_SUB documents each, so the sub-batch is the slot; 65536 keeps the serial schedule (a paired CTA would hold one
    warp and cut emit's residency)"""
    n = 2 * PAIR_SUB if cls == 17408 else 60_000
    arena, offs, lens = W.chat_corpus(17, 0, n, target=1024)
    paired, serial = both_schedules(ctx, ctx.cfg("aws-bedrock"), arena, offs, lens, max_len=cls)
    recs, res, launches = paired
    if cls == 65536:
        assert launches % 4 == 0 and launches >= 8, launches
        assert recs == serial[0]
    else:
        assert check_paired(paired, serial, n) >= 3
    assert (res["status"] == OK).all()
    oracle_sample("aws-bedrock", arena, offs, lens, recs, range(0, n, 499))


def packed(bodies):
    import aigw_b200 as A
    return A.capi.pack_bodies(bodies)


@pytest.fixture(scope="module")
def diverse():
    """4096 bodies of the diverse corpus (accepted, declined and 400 bodies interleaved), repeated past one sub-batch"""
    base = [W.diverse_body(s) for s in range(4096)]
    n = 2 * PAIR_SUB + 4096 + 17
    return packed([base[i % len(base)] for i in range(n)])


@pytest.mark.parametrize("schema,override", [("openai", "override-model"), ("gcp-vertexai", None), ("gcp-anthropicai", None), ("resp-error-aws-bedrock", None)])
def test_diverse_schemas(ctx, diverse, schema, override):
    arena, offs, lens = diverse
    n = len(lens)
    paired, serial = both_schedules(ctx, ctx.cfg(schema, model_override=override), arena, offs[:n], lens)
    check_paired(paired, serial, n)
    assert (paired[1]["status"] == OK).any()
    if schema == "openai":
        oracle_sample(schema, arena, offs, lens, paired[0], boundaries(3, n, step=211), model_override=override)


def test_response_schema(ctx):
    """buffered Bedrock Converse responses (the response id table of the index stage)"""
    rng = np.random.default_rng(23)
    base = [W.bedrock_response_body(rng, ["plain", "tools", "reasoning", "cache"][i % 4]) for i in range(2048)]
    n = 2 * PAIR_SUB + 2048 + 3
    arena, offs, lens = packed([base[i % len(base)] for i in range(n)])
    paired, serial = both_schedules(ctx, ctx.cfg("resp-aws-bedrock", model_override="m"), arena, offs[:n], lens)
    check_paired(paired, serial, n)
    assert (paired[1]["status"] == OK).mean() > 0.9


def test_device_mapped(ctx):
    """aigw_chat_translate_device_mapped: sub-batches are cut from the document map, not from the document numbers"""
    n = 2 * PAIR_SUB + 3000
    arena, offs, lens = W.chat_corpus(19, 0, n, target=1500)
    doc_map = np.random.default_rng(5).permutation(n).astype(np.uint32)
    paired, serial = both_schedules(ctx, ctx.cfg("aws-bedrock"), arena, offs, lens, doc_map=doc_map)
    check_paired(paired, serial, n)
    assert (paired[1]["status"] == OK).all()
    oracle_sample("aws-bedrock", arena, offs, lens, paired[0], [int(doc_map[i]) for i in boundaries(3, n)])
