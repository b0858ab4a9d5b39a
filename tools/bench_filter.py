"""Filtered search on one GPU (DESIGN.md 3.6): filter build time and bytes, filtered against unfiltered QPS (device-resident, CUDA events
after a warm-up, as bench.py times its search), the share of probed code blocks the scan skips, 16 queries per filter checked bit for
bit against the CPU oracle (lists regenerated from the seed), and the post-filter baseline: an unfiltered search with
k' = min(1024, 2 ceil(k / selectivity)), cut to the selected labels, and the share of queries whose filtered top-k it reproduces.

    python tools/bench_filter.py [--workloads C2 C4] [--steps K] [--warmup W] [--out DIR]

Workloads: C2 (100 M rows, IVF4096, batch 64, nprobe 256, k 10) and C4's shape on one GPU (500 M rows, IVF65536, batch 1024, nprobe 32
and 256, k 10), synthetic lists and bench.py's near queries.  Filters: random label sets of 50 %, 10 % and 1 % of the labels, a range
of 1 M labels, the exclude form of the 1 % set, and everything selected.  Prints one JSON document (written to DIR when --out is given).
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload shapes, seeds and the query plan of the flagship benchmark)

SPECS = {"C2": dict(N=100_000_000, nlist=4096, batch=64, nprobes=(256,)),
         "C4": dict(N=500_000_000, nlist=65536, batch=1024, nprobes=(32, 256))}
K = 10


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip()


def random_labels(N, pct, seed):
    """A pct % random subset of 0 .. N-1 (sorted), drawn in chunks."""
    rng = np.random.default_rng(seed)
    parts = []
    for a in range(0, N, 1 << 26):
        b = min(N, a + (1 << 26))
        parts.append(a + np.flatnonzero(rng.random(b - a) < pct / 100.0))
    return np.concatenate(parts).astype(np.int64)


def filters(N):
    one = random_labels(N, 1, 3)
    lo = N // 3
    return {"set50": (random_labels(N, 50, 1), False), "set10": (random_labels(N, 10, 2), False), "set1": (one, False),
            "range1M": (range(lo, lo + 1_000_000), False), "set1_exclude": (one, True), "everything": (np.zeros(0, np.int64), True)}


def selected_of(sel, exclude, N):
    """bool [N]: the selected rows of a sequential-label index (label = list-major row)."""
    s = np.zeros(N, bool)
    if isinstance(sel, range):
        s[sel.start:sel.stop] = True
    else:
        s[sel] = True
    return s != exclude


def timed(ix, Q, W, Kst, flt):
    import torch
    for s in range(W):
        ix.search(Q[s], K, filter=flt)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = None
    for s in range(W, W + Kst):
        out = ix.search(Q[s], K, filter=flt)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def skipped_share(ix, lens, mask, n):
    """Share of the probed (query, code block) pairs whose mask word is 0, from the last batch's probes."""
    nb = (lens + 31) // 32
    boff = np.concatenate([[0], np.cumsum(nb)])
    empty_per_list = np.add.reduceat(mask == 0, boff[:-1]) * (nb > 0) if len(mask) else np.zeros(len(lens))
    probes = ix.last_probes(n).ravel()
    probes = probes[probes >= 0]
    return float(empty_per_list[probes].sum() / max(nb[probes].sum(), 1))


def run(name, W, Kst, oracle):
    import torch
    from densephrases_b200 import IvfPqIndex
    from oracle import filter_ref as FR
    sp = SPECS[name]
    N, nlist, B = sp["N"], sp["nlist"], sp["batch"]
    wl = dict(name=name, N=N, nlist=nlist, batch=B, nprobe=sp["nprobes"][0], k=K, lens=bench.uniform_lens(N, nlist))
    lens = wl["lens"]
    A = bench.opq_matrix(bench.SEED_INDEX)
    ix = IvfPqIndex(nlist)
    ix.set_opq(A); ix.gen_centroids(bench.SEED_INDEX); ix.gen_pq(bench.SEED_INDEX)
    ix.set_lists_synthetic(lens, bench.SEED_INDEX)
    torch.cuda.synchronize()
    ids, noise = bench.make_query_plan(wl, W + Kst)
    v, _ = ix.reconstruct_batch(ids.cuda())
    Qh = bench.finish_queries(v.cpu(), noise, A).reshape(W + Kst, B, bench.D)
    Q = Qh.cuda()
    ref = bench.ref_index_for(wl, oracle)
    res = {"workload": f"{name}: {N} rows, IVF{nlist}, batch {B}, k {K}", "device_bytes": ix.device_bytes, "nprobe": {}}
    built = {}
    for fname, (sel, exclude) in filters(N).items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f = ix.make_filter(torch.from_numpy(sel).cuda() if isinstance(sel, np.ndarray) else sel, exclude=exclude)
        ms = (time.perf_counter() - t0) * 1e3
        built[fname] = (f, selected_of(sel, exclude, N))
        res.setdefault("filters", {})[fname] = {"rows": f.rows, "selectivity": f.rows / N, "bytes": f.nbytes, "build_ms": ms}
    for nprobe in sp["nprobes"]:
        ix.nprobe = nprobe
        ms0, (D0, I0) = timed(ix, Q, W, Kst, None)
        r = {"unfiltered_qps": B * Kst / (ms0 / 1e3), "filters": {}}
        xq = Qh[W + Kst - 1][:16].numpy()
        rr = ref.with_resident_lists(np.unique(ref.coarse(ref.rotate(xq), nprobe)[1]))
        for fname, (f, selected) in built.items():
            ms, (D, I) = timed(ix, Q, W, Kst, f)
            D, I = D.cpu().numpy(), I.cpu().numpy()
            skip = skipped_share(ix, lens, f.mask(), B)
            Dr, Ir, _ = FR.search(rr, xq, K, nprobe, selected.astype(np.uint8))
            ok = bool(np.array_equal(D[:16].view(np.int32), Dr.view(np.int32)) and np.array_equal(I[:16], Ir))
            kp = min(1024, 2 * math.ceil(K / max(f.rows / N, 1e-12)))
            _, Ip = ix.search(Q[W + Kst - 1], kp)
            Ip = Ip.cpu().numpy()
            hit = 0
            for qi in range(B):
                lab = Ip[qi][Ip[qi] >= 0]
                kept = lab[selected[lab]][:K]
                want = I[qi][I[qi] >= 0]
                hit += int(len(kept) == len(want) and np.array_equal(kept, want))
            r["filters"][fname] = {"qps": B * Kst / (ms / 1e3), "vs_unfiltered": ms0 / ms, "skipped_block_share": skip,
                                   "oracle_16_bit_identical": ok, "postfilter_k": kp, "postfilter_reproduces": hit / B}
        res["nprobe"][str(nprobe)] = r
        del D0, I0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["C2", "C4"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_filter: needs a GPU")
    from oracle import ivfpq_ref as oracle
    oracle.build()
    bench.oracle_threads(oracle)
    out = {"gpu": card(), "steps": args.steps, "warmup": args.warmup, "results": {}}
    for name in args.workloads:
        out["results"][name] = run(name, args.warmup, args.steps, oracle)
        torch.cuda.empty_cache()
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_filter.json"), "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
