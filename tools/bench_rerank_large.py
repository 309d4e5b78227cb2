"""Throughput and latency of aigw_rerank_translate_large_* on the large realistic rerank corpus (tests/test_rerank_large_cpu.py:
300 RAG reranks of 64 KiB to 8 MiB, about 83 MB).  Prints one JSON line; --out also writes it to a file.

  device      the device call on device-resident bodies, without and with the model override: bodies/s, GB/s of request plus
              output bytes, whole-call CUDA-event time, and the scan / emit kernel times from torch.profiler (a separate pass)
  host        the host call end to end (H2D, kernels, D2H of the records)
  latency     one request per host call, wall clock p50 / p99, at 128 KiB, 1 MiB and 4 MiB
  serial walk the worst case of the scan's one-thread member walk: 16 MiB - 1 bodies holding the most tokens a request may
              (len / 4 + 1024), in an unknown member's value, or in a documents array with one object element (both walked by
              one thread), against the same tokens in a flat documents array (checked in parallel)
  oracle      the Python restatement (tests/_rerank_oracle.py), one thread, on a sample: the CPU yardstick, not the Go reference

usage: python tools/bench_rerank_large.py [--reps 20] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, clk = [x.strip() for x in q.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the number is still reported, the card is then unknown
        return {"gpu": "unknown (%s)" % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    import aigw_b200 as A
    import _rerank_oracle as Q
    import test_rerank_large_cpu as L
    ctx = A.Context(0)
    res = {"card": card(), "workload": "test_rerank_large_cpu.large_corpus(): 300 Cohere /v2/rerank requests, 64 KiB - 8 MiB"}
    bodies = L.large_corpus()
    arena, offs, lens = A.pack_bodies(bodies)
    n, in_bytes = len(bodies), int(lens.sum())
    res["bodies"], res["request_bytes"] = n, in_bytes
    cap = int(sum((len(b) + 200 + 15) // 16 * 16 for b in bodies))
    d_b, d_o, d_l, d_out, d_r, d_u = (ctx.dalloc(max(16, x)) for x in (arena.nbytes, offs.nbytes, lens.nbytes, cap, n * 32, 8))
    ctx.h2d(d_b, arena); ctx.h2d(d_o, offs); ctx.h2d(d_l, lens)
    used = np.zeros(1, dtype=np.uint64)
    for label, override in (("device_no_override", ""), ("device_override", "rerank-v3.5")):
        c = ctx.cfg("rerank-cohere", model_override=override or None, api_version="v2")
        ms = []
        for rep in range(a.reps + 3):
            ctx.memset(d_u, 0, 8)
            t = ctx.rerank_translate_large_device(c, d_b, d_o, d_l, n, int(lens.max()), d_out, cap, d_r, d_u)
            if rep >= 3:
                ms.append(t)
        ctx.d2h(used, d_u)
        med = float(np.median(ms))
        moved = in_bytes + int(used[0])
        res[label] = {"call_ms_median": med, "call_ms_min": float(min(ms)), "bodies_per_s": n / med * 1e3, "GB_per_s_in_plus_out": moved / med / 1e6,
                      "output_bytes": int(used[0])}
        # per-kernel times in a profiled pass of its own
        try:
            import torch
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    ctx.memset(d_u, 0, 8)
                    ctx.rerank_translate_large_device(c, d_b, d_o, d_l, n, int(lens.max()), d_out, cap, d_r, d_u)
            k = {}
            for e in prof.key_averages():
                for name in ("rerank_scan_kernel", "rerank_emit_kernel"):
                    if name in e.key:
                        k[name + "_ms"] = e.device_time_total / 1e3 / 5 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3 / 5
            res[label].update(k)
        except Exception as e:
            res[label]["kernel_split"] = "not measured (%s)" % e
    for d in (d_b, d_o, d_l, d_out, d_r, d_u):
        ctx.dfree(d)
    # the host call end to end
    c = ctx.cfg("rerank-cohere", model_override="rerank-v3.5", api_version="v2")
    wall = []
    for rep in range(max(3, a.reps // 4) + 1):
        t0 = time.perf_counter()
        r, out, st = ctx.rerank_translate_large_host(c, arena, offs, lens)
        if rep:
            wall.append((time.perf_counter() - t0) * 1e3)
    assert (r["status"] == 0).all()
    med = float(np.median(wall))
    res["host_override"] = {"wall_ms_median": med, "bodies_per_s": n / med * 1e3, "GB_per_s_request": in_bytes / med / 1e6, "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"]}
    # single-request latency
    lat = {}
    for size in (128 << 10, 1 << 20, 4 << 20):
        b = L.sized_body(size, seed=size)
        a1, o1, l1 = A.pack_bodies([b])
        ts = []
        for rep in range(a.reps * 5 + 5):
            t0 = time.perf_counter()
            ctx.rerank_translate_large_host(c, a1, o1, l1)
            if rep >= 5:
                ts.append((time.perf_counter() - t0) * 1e6)
        lat["%d_KiB" % (size >> 10)] = {"p50_us": float(np.percentile(ts, 50)), "p99_us": float(np.percentile(ts, 99)), "samples": len(ts)}
    res["single_request_latency_host_call"] = lat
    # the serial member walk at its worst: every token a request may hold, walked by one thread
    n16 = (16 << 20) - 1
    cap16 = n16 // 4 + 1024 - 64

    def exact(head, mid, tail=b'],"pad":"', end=b'"}'):
        body = head + mid + tail
        return body + b"x" * (n16 - len(body) - len(end)) + end

    k2, k3 = cap16 // 2 - 16, cap16 // 3 - 16
    worst = {
        "unknown_member_value": (exact(b'{"model":"m","metadata":[', b"0," * (k2 - 1) + b"0"), 0),
        "documents_with_an_object_element": (exact(b'{"model":"m","documents":[{},', b'"",' * (k3 - 1) + b'""'), 1),
        "flat_documents_same_tokens": (exact(b'{"model":"m","documents":[', b'"",' * k3 + b'""'), 0),
    }
    walk = {}
    c0 = ctx.cfg("rerank-cohere", api_version="v2")
    for name, (b, want) in worst.items():
        a1, o1, l1 = A.pack_bodies([b])
        ks = []
        for rep in range(4):
            r1, _, st = ctx.rerank_translate_large_host(c0, a1, o1, l1)
            if rep:
                ks.append(st["kernel_ms"])
        walk[name] = {"bytes": len(b), "scan_tokens_about": cap16, "kernel_ms_median": float(np.median(ks)), "status": int(r1[0]["status"]),
                      "reason": int(r1[0]["reason"]), "expected_status": want}
    res["serial_walk_worst_case"] = walk
    # the Python oracle, one thread
    sample = bodies[4:34]
    t0 = time.perf_counter()
    for b in sample:
        Q.parse_body(b)
    dt = time.perf_counter() - t0
    sb = sum(len(b) for b in sample)
    res["python_oracle_one_thread"] = {"bodies": len(sample), "bytes": sb, "MB_per_s": sb / dt / 1e6, "note": "CPU restatement used by the tests, not the Go reference"}
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
