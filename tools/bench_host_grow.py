"""Mutable host indexes (DESIGN.md 3.5, "Mutable host indexes") on one GPU: add, remove and merge in place on a page-locked code array.

  python tools/bench_host_grow.py [--legs c2,build,reserve] [--build-max-rows N] [--out DIR]

c2:      a C2-shaped host index (100 M rows, IVF4096, 9.6 GB of codes, synthetic) with a reserved capacity: add 1 M rows, remove a
         1 M-label range, merge a 10 M-row device-resident source.  Each call: time, blocks the mover read and wrote, its rate, and
         the device-resident twin's time for the same call.  Reference rates: cudaMemcpyAsync host-to-device and device-to-host
         of 1 GiB from page-locked memory, alone and both directions at once.
build:   an empty host index grown by adds of 10 M rows (one device batch, reused) up to the largest multiple of 10 M rows whose codes
         fit 60 % of MemAvailable (capped by --build-max-rows): time per add against rows held.
reserve: the growth copy of reserve_host_codes (a larger page-locked array, the codes copied over).
Every leg checks 64 queries bit for bit against a device-resident twin where one is kept.  Prints one JSON document (also written to
DIR/host_grow.json with --out) with the card name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (seeds and workloads shared with the benchmark)
from densephrases_b200 import IvfPqIndex  # noqa: E402
from tools.bench_host_codes import card, mem_available  # noqa: E402

GiB = 1 << 30
SEED = bench.SEED_INDEX


def make(lens, nlist, on_host, capacity=0, seed=SEED):
    ix = IvfPqIndex(nlist)
    ix.set_opq(bench.opq_matrix(SEED))
    ix.gen_centroids(SEED)
    ix.gen_pq(SEED)
    if on_host:
        ix.set_code_residency(True, 2 * GiB)
        ix.reserve_host_codes(capacity)
    ix.set_lists_synthetic(lens, seed)
    return ix


def batch(ix, n, seed):
    """n vectors near random centroids, on the device (rotated back through the OPQ matrix)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = torch.from_numpy(ix.centroids()).cuda()
    A = torch.from_numpy(ix.opq_matrix()).cuda()
    out = torch.empty((n, 768), dtype=torch.float32, device="cuda")
    for o in range(0, n, 1 << 20):
        m = min(1 << 20, n - o)
        idx = torch.randint(0, C.shape[0], (m,), device="cuda", generator=g)
        out[o:o + m] = (C[idx] + 0.3 * torch.randn((m, 768), device="cuda", generator=g)) @ A
    return out


def same_bits(ix, twin, q, nprobe=64):
    for g in (ix, twin):
        g.nprobe = nprobe
    D, I = ix.search(q, 10)
    Dt, It = twin.search(q, 10)
    return bool(np.array_equal(D.view(np.int32), Dt.view(np.int32)) and np.array_equal(I, It))


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def copy_rates(nbytes=GiB):
    """cudaMemcpyAsync GB/s from / to page-locked memory: H2D, D2H, and both at once on two streams (best of 3)."""
    import torch
    h = [torch.empty(nbytes, dtype=torch.uint8).pin_memory() for _ in range(2)]
    d = [torch.empty(nbytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
    s = [torch.cuda.Stream() for _ in range(2)]
    best = {"h2d": 0.0, "d2h": 0.0, "both_each_way": 0.0}
    for _ in range(3):
        ms, _ = timed(lambda: d[0].copy_(h[0], non_blocking=True))
        best["h2d"] = max(best["h2d"], nbytes / ms / 1e6)
        ms, _ = timed(lambda: h[1].copy_(d[1], non_blocking=True))
        best["d2h"] = max(best["d2h"], nbytes / ms / 1e6)

        def both():
            with torch.cuda.stream(s[0]):
                d[0].copy_(h[0], non_blocking=True)
            with torch.cuda.stream(s[1]):
                h[1].copy_(d[1], non_blocking=True)
        ms, _ = timed(both)
        best["both_each_way"] = max(best["both_each_way"], nbytes / ms / 1e6)
    return {k: round(v, 1) for k, v in best.items()}


def c2_leg():
    import torch
    wl = bench.workload("C2")
    lens, nlist = wl["lens"], wl["nlist"]
    nb = int(((lens + 31) // 32).sum())
    out = {"rows": int(lens.sum()), "codes_GB": nb * 3072 / 1e9, "copy_engine_GBps": copy_rates()}
    capacity = (nb + 2 * 1_000_000 // 32 + 2 * 10_000_000 // 32 + 2 * nlist) * 3072
    ix = make(lens, nlist, True, capacity)
    twin = make(lens, nlist, False)
    out["host_bytes"] = ix.host_bytes
    q = batch(ix, 64, 5).cpu().numpy()
    out["bits_equal_before"] = same_bits(ix, twin, q)
    src_lens = np.random.default_rng(3).multinomial(10_000_000, np.full(nlist, 1 / nlist)).astype(np.int64)
    src = make(src_lens, nlist, False, seed=SEED + 1)
    x = batch(ix, 1_000_000, 100)
    calls = {
        "add_1M": lambda g: g.add(x),
        "remove_1M_range": lambda g: g.remove_ids(range(40_000_000, 41_000_000)),
        "merge_10M_source": lambda g: g.merge_from(src, add_id=10**9),
    }
    for name, call in calls.items():
        ms, _ = timed(lambda: call(ix))
        mv = ix.last_host_move()
        tms, _ = timed(lambda: call(twin))
        rd, wr = mv["blocks_read"] * 3072, mv["blocks_written"] * 3072
        r = {"ms": round(ms, 1), "mover_ms": round(mv["ms"], 1), "GB_read": round(rd / 1e9, 2), "GB_written": round(wr / 1e9, 2),
             "chunks": mv["chunks"], "mover_GBps_each_way": round(max(rd, wr) / max(mv["ms"], 1e-3) / 1e6, 1),
             "device_twin_ms": round(tms, 1), "bits_equal": same_bits(ix, twin, q)}
        out[name] = r
        print("c2", name, r, flush=True)
    out["host_bytes_after"] = ix.host_bytes
    del ix, twin, src, x
    torch.cuda.empty_cache()
    return out


def build_leg(max_rows):
    import torch
    nlist, step = 4096, 10_000_000
    rows = min(max_rows, int(0.6 * mem_available() / 96) // step * step)
    out = {"mem_available_GB": round(mem_available() / 1e9, 1), "target_rows": rows, "adds": []}
    if rows < step:
        out["note"] = "not measured: host memory"
        return out
    cap = (rows // 32 + 2 * nlist) * 3072
    ix = make(np.zeros(nlist, np.int64), nlist, True, cap)
    twin = make(np.zeros(nlist, np.int64), nlist, False)
    x = batch(ix, step, 7)
    q = batch(ix, 64, 8).cpu().numpy()
    twin_rows = 100_000_000
    while ix.ntotal + step <= rows:
        ms, _ = timed(lambda: ix.add(x))
        mv = ix.last_host_move()
        rec = {"rows_held": ix.ntotal, "ms": round(ms, 1), "mover_ms": round(mv["ms"], 1), "GB_written": round(mv["blocks_written"] * 3072 / 1e9, 2)}
        if twin is not None:
            twin.add(x)
            if twin.ntotal == twin_rows:
                rec["bits_equal"] = same_bits(ix, twin, q)
                del twin
                twin = None
                torch.cuda.empty_cache()
        out["adds"].append(rec)
        print("build", rec, flush=True)
    out["rows"] = ix.ntotal
    out["host_bytes"] = ix.host_bytes
    del ix
    torch.cuda.empty_cache()
    return out


def reserve_leg():
    wl = bench.workload("C2")
    ix = make(wl["lens"], wl["nlist"], True, 0)
    twin = make(wl["lens"], wl["nlist"], False)
    before = ix.host_bytes
    ms, _ = timed(lambda: ix.reserve_host_codes(before + 2 * GiB))
    q = batch(ix, 64, 9).cpu().numpy()
    return {"from_bytes": before, "to_bytes": ix.host_bytes, "ms": round(ms, 1), "copy_GBps": round(before / ms / 1e6, 1),
            "bits_equal": same_bits(ix, twin, q)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="c2,build,reserve")
    ap.add_argument("--build-max-rows", type=int, default=300_000_000)
    ap.add_argument("--out", default=None, help="also write DIR/host_grow.json")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_host_grow: no GPU (there is no CPU fallback)")
    res = {"card": card()}
    print(res, flush=True)
    legs = a.legs.split(",")
    if "c2" in legs:
        res["c2"] = c2_leg()
    if "reserve" in legs:
        res["reserve"] = reserve_leg()
        print("reserve", res["reserve"], flush=True)
    if "build" in legs:
        res["build"] = build_leg(a.build_max_rows)
    res["card_after"] = card()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "host_grow.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
