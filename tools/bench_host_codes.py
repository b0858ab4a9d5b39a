"""Codes in host memory (DESIGN.md 3.5) on one GPU: fetch rate, C4 with the full index, C2 resident vs host mode.

  python tools/bench_host_codes.py [--legs fetch,c4,c2] [--c4-rows N] [--out DIR]

fetch: fetch_lists_kernel (timed as set_resident_lists of every list: the gather from mapped host memory, plus the region's
       allocation) against cudaMemcpyAsync host-to-device of the same bytes from a page-locked buffer (the copy-engine reference),
       for ~53 KB lists (C5-like) and ~1.46 MB lists (C4), about 8 GB each.
c4:    IVF65536, batch 1024, k 10, nprobe 32 and 256, 16 GiB stream region, 1 B phrases (or the largest multiple of 100 M whose codes
       fit 80 % of MemAvailable page-locked); resident sets: none, and the most-probed lists of a separate query sample that fit the
       HBM left; QPS, GB fetched, fetch ms, scan ms and slices per batch; 16 queries of the last batch checked bit for bit against
       the CPU oracle (lists regenerated from the seed).
c2:    100 M phrases, IVF4096, batch 64, nprobe 256: device-resident index vs host mode with every list resident vs none.
Prints one JSON document (also written to DIR/host_codes.json with --out) with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (seeds, workloads and query plan shared with the benchmark)
from densephrases_b200 import IvfPqIndex  # noqa: E402

GiB = 1 << 30


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return out


def mem_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def synthetic(lens, nlist, stream_bytes, on_host=True):
    ix = IvfPqIndex(nlist)
    ix.set_opq(bench.opq_matrix(bench.SEED_INDEX))
    ix.gen_centroids(bench.SEED_INDEX)
    ix.gen_pq(bench.SEED_INDEX)
    if on_host:
        ix.set_code_residency(True, stream_bytes)
    ix.set_lists_synthetic(lens, bench.SEED_INDEX)
    return ix


def fetch_leg():
    import torch
    out = {}
    for name, rows in (("53KB_lists", 553), ("1.46MB_lists", 15259)):
        blocks = (rows + 31) // 32
        nlist = int(8e9 // (blocks * 3072))
        nbytes = nlist * blocks * 3072
        ix = synthetic(np.full(nlist, rows, np.int64), nlist, 0)
        torch.cuda.synchronize()
        ts = []
        for _ in range(3):
            ix.set_resident_lists([])
            t0 = time.perf_counter()
            ix.set_resident_lists(np.arange(nlist))
            ts.append(time.perf_counter() - t0)
        ix.set_resident_lists([])
        del ix
        h = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
        d = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ce = []
        for _ in range(3):
            e0.record()
            d.copy_(h, non_blocking=True)
            e1.record()
            torch.cuda.synchronize()
            ce.append(e0.elapsed_time(e1) / 1e3)
        del h, d
        torch.cuda.empty_cache()
        fk, cp = nbytes / min(ts) / 1e9, nbytes / min(ce) / 1e9
        out[name] = {"lists": nlist, "bytes": nbytes, "fetch_kernel_GBps": fk, "copy_engine_GBps": cp, "ratio": fk / cp,
                     "note": "best of 3; fetch includes the region's cudaMalloc"}
        print(name, out[name], flush=True)
    return out


def probe_counts(ix, q, nlist):
    ix.search(q, 10)
    keys = ix.last_probes(len(q)).ravel()
    return np.bincount(keys[keys >= 0], minlength=nlist)


def run_batches(ix, Q, k, steps):
    """-> per-batch means over `steps` timed batches (after one warm-up), then one profiled batch for fetch and scan times."""
    ix.set_profile(False)
    ix.search(Q[0], k)
    t, fetched, slices = [], [], []
    for b in range(steps):
        t0 = time.perf_counter()
        D, I = ix.search(Q[1 + b], k)
        t.append(time.perf_counter() - t0)
        f = ix.last_fetch()
        fetched.append(f["blocks_fetched"] * 3072 / 1e9); slices.append(f["slices"])
    ix.set_profile(True)
    ix.search(Q[1], k)
    f = ix.last_fetch()
    scan = float(ix.profile_scan_ms()[-f["slices"]:].sum()) if f["slices"] <= 64 else None
    ix.set_profile(False)
    n = Q[0].shape[0]
    return {"qps": n / float(np.mean(t)), "batch_s": float(np.mean(t)), "GB_fetched_per_batch": float(np.mean(fetched)),
            "slices_per_batch": float(np.mean(slices)), "fetch_ms_profiled": f["fetch_ms"], "scan_ms_profiled": scan,
            "fetch_GBps_profiled": f["blocks_fetched"] * 3072 / 1e9 / (f["fetch_ms"] / 1e3) if f["fetch_ms"] else None}, (D, I)


def queries(ix, wl, nb, offset=0):
    ids, noise = bench.make_query_plan(wl, nb + offset)
    v, _ = ix.reconstruct_batch(ids.numpy())
    import torch
    q = bench.finish_queries(torch.from_numpy(v), noise, bench.opq_matrix(bench.SEED_INDEX)).numpy()
    return [q[i * wl["batch"]:(i + 1) * wl["batch"]] for i in range(offset, offset + nb)]


def oracle_check(wl, nprobe, Q, res):
    from oracle import ivfpq_ref as oracle
    oracle.build()
    bench.oracle_threads(oracle)
    ref = bench.ref_index_for(wl, oracle)
    pick = np.arange(0, wl["batch"], wl["batch"] // 16)[:16]
    Dr, Ir = ref.search(Q[pick], wl["k"], nprobe)
    D, I = res[0][pick], res[1][pick]
    return {"queries": 16, "identical_ids_and_fp32_scores": bool(np.array_equal(D.view(np.int32), Dr.view(np.int32)) and np.array_equal(I, Ir))}


def c4_leg(rows, steps):
    import torch
    avail = mem_available()
    N = rows or 1_000_000_000
    while N > 100_000_000 and N * 96 > 0.8 * avail:
        N -= 100_000_000
    wl = bench.workload("C4", N / 1e9)
    note = f"{N} phrases ({N * 96 / 1e9:.0f} GB of codes page-locked; MemAvailable {avail / 1e9:.0f} GB)"
    print("c4:", note, flush=True)
    t0 = time.perf_counter()
    ix = synthetic(wl["lens"], wl["nlist"], 16 * GiB)
    build_s = time.perf_counter() - t0
    Q = queries(ix, wl, steps + 1)
    sample = queries(ix, wl, 1, offset=steps + 1)[0]
    out = {"phrases": N, "note": note, "build_s": build_s, "host_bytes": ix.host_bytes}
    for nprobe in (32, 256):
        ix.nprobe = nprobe
        counts = probe_counts(ix, sample, wl["nlist"])
        for res_name in ("none", "most_probed"):
            ix.set_resident_lists([])
            res = []
            if res_name == "most_probed":
                # the new region (resident + stream) is allocated while the old one lives; keep the batch workspace free
                budget = torch.cuda.mem_get_info()[0] - 16 * GiB - 6 * GiB
                per = (wl["lens"] + 31) // 32 * 3072
                order = np.argsort(-counts, kind="stable")
                res = order[np.cumsum(per[order]) <= budget]
                ix.set_resident_lists(res)
            r, last = run_batches(ix, Q, wl["k"], steps)
            r.update(resident_lists=int(len(res)), device_bytes=ix.device_bytes)
            r["oracle_check"] = oracle_check(wl, nprobe, Q[steps], last) if res_name == "none" else None
            out[f"nprobe{nprobe}_resident_{res_name}"] = r
            print(nprobe, res_name, r, flush=True)
    del ix
    torch.cuda.empty_cache()
    return out


def c2_leg(steps):
    import torch
    wl = bench.workload("C2")
    out = {}
    for name in ("device", "host_all_resident", "host_none_resident"):
        on_host = name != "device"
        ix = synthetic(wl["lens"], wl["nlist"], 2 * GiB if on_host else 0, on_host)
        if name == "host_all_resident":
            ix.set_resident_lists(np.arange(wl["nlist"]))
        ix.nprobe = wl["nprobe"]
        Q = queries(ix, wl, steps + 1)
        ix.search(Q[0], wl["k"])
        t0 = time.perf_counter()
        for b in range(steps):
            ix.search(Q[1 + b], wl["k"])
        dt = (time.perf_counter() - t0) / steps
        r = {"qps": wl["batch"] / dt, "batch_ms": dt * 1e3}
        if on_host:
            f = ix.last_fetch()
            r.update(slices=f["slices"], GB_fetched=f["blocks_fetched"] * 3072 / 1e9)
        out[name] = r
        print("c2", name, r, flush=True)
        del ix
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="fetch,c4,c2")
    ap.add_argument("--c4-rows", type=int, default=0, help="phrases of the C4 leg (0: 1 B, or what fits host memory)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write DIR/host_codes.json")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_host_codes: no GPU (there is no CPU fallback)")
    res = {"card": card()}
    print(res, flush=True)
    legs = a.legs.split(",")
    if "fetch" in legs:
        res["fetch"] = fetch_leg()
    if "c4" in legs:
        res["c4"] = c4_leg(a.c4_rows, a.steps)
    if "c2" in legs:
        res["c2"] = c2_leg(20)
    res["card_after"] = card()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "host_codes.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
