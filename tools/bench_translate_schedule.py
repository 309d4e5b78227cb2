"""Paired vs serial schedule of the device translate call on bench.py's config-2 workload (1 M bodies of ~4 KB, OpenAI -> AWS
Bedrock Converse, device-resident inputs).  The default call runs the paired schedule (index of sub-batch k+1 beside the emit of
sub-batch k); with the stage profile on (aigw_chat_set_profile) the same call runs the serial schedule.  The two alternate in one
process, each timed by the library's CUDA events, and their results are compared per document.

    python tools/bench_translate_schedule.py [--bodies 1000000] [--rounds 5] [--calls 3] [--out DIR]

Prints one JSON line: ms per call (median, min, max over rounds) for each schedule, the card's name, power limit and SM clock,
and whether every document's result and record bytes match."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SEED = 2   # bench.py config 2
FIELDS = ("status", "reason", "body_len", "path_len", "body_kind", "flags", "model_off", "model_len")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bodies", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the two schedules")
    ap.add_argument("--calls", type=int, default=3, help="timed calls per schedule per round")
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import aigw_b200 as A
    import _workload as W
    A.load_library()
    ctx = A.Context(0)
    n = a.bodies
    lens = W.chat_lens(SEED, 0, n)
    offs = W.chat_offsets(lens)
    in_bytes = int(offs[-1]) + 16
    src = np.full(in_bytes, 0x20, dtype=np.uint8)
    W.chat_fill(SEED, 0, n, src, offs, lens)
    max_len = int(lens.max())
    cfg = ctx.cfg("aws-bedrock")
    d_in = ctx.dalloc(in_bytes); d_off = ctx.dalloc(offs.nbytes); d_len = ctx.dalloc(lens.nbytes)
    out_cap = int(in_bytes * 1.25) + n * 64 + 4096
    d_out = ctx.dalloc(out_cap); d_res = ctx.dalloc(n * 32); d_used = ctx.dalloc(8)
    ctx.h2d(d_in, src); ctx.h2d(d_off, offs); ctx.h2d(d_len, lens)

    def call(serial):
        ctx.chat_set_profile(serial)
        try:
            ctx.memset(d_used, 0, 8)
            ms = ctx.chat_translate_device(cfg, d_in, d_off, d_len, n, max_len, d_out, out_cap, d_res, d_used)
            return ms, ctx.chat_last_profile()["launches"]
        finally:
            ctx.chat_set_profile(False)

    def outputs():
        res = np.zeros(n, dtype=A.DocResult); ctx.d2h(res, d_res)
        used = np.zeros(1, dtype=np.uint64); ctx.d2h(used, d_used)
        out = np.zeros(max(16, int(used[0])), dtype=np.uint8); ctx.d2h(out, d_out, int(used[0]))
        # records in document order (out_off is where the bump allocator put them, which depends on completion order)
        ok = res["status"] == A.AIGW_OK
        o = res["out_off"].astype(np.int64); ln = res["path_len"].astype(np.int64) + res["body_len"].astype(np.int64)
        recs = np.concatenate([out[o[i]:o[i] + ln[i]] for i in np.nonzero(ok)[0]]) if ok.any() else np.zeros(0, np.uint8)
        return {f: res[f].copy() for f in FIELDS}, recs

    for _ in range(a.warmup):
        call(False); call(True)
    times = {"paired": [], "serial": []}; launches = {}
    for _ in range(a.rounds):
        for name, serial in (("paired", False), ("serial", True)):
            ms = []
            for _ in range(a.calls):
                t, launches[name] = call(serial)
                ms.append(t)
            times[name].append(float(np.median(ms)))
    call(False); pr, prec = outputs()
    call(True); sr, srec = outputs()
    same = all(np.array_equal(pr[f], sr[f]) for f in FIELDS) and np.array_equal(prec, srec)
    for p in (d_in, d_off, d_len, d_out, d_res, d_used):
        ctx.dfree(p)
    ctx.close()
    summ = {k: {"ms_median": float(np.median(v)), "ms_min": float(np.min(v)), "ms_max": float(np.max(v)), "rounds": v, "launches": launches[k]} for k, v in times.items()}
    print(json.dumps({"bodies": n, "max_len": max_len, "chat_sub_env": os.environ.get("AIGW_CHAT_SUB"), "schedules": summ,
                      "speedup_median": summ["serial"]["ms_median"] / summ["paired"]["ms_median"], "per_document_equal": bool(same), "card": card()}))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
