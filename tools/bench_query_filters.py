"""Per-query filters on one GPU (DESIGN.md 3.7): build time of make_query_filters against the sum of make_filter over the same selectors,
the filter's bytes, QPS (device-resident queries, CUDA events after a warm-up, as bench_filter.py), the fast pass's scan kernel time, the
selected blocks read as a share of the probed blocks, and 16 sampled queries checked bit for bit against the CPU oracle (lists
regenerated from the seed).  The baseline is the only way without per-query filters: a loop of one-query searches with each query's
make_filter, prebuilt (where the masks fit) and built in the loop.

    python tools/bench_query_filters.py [--workloads C2 C4] [--steps K] [--warmup W] [--loop-queries Q] [--out DIR]

Workloads: C2 (100 M rows, IVF4096, batch 64, nprobe 256) and C4's shape on one GPU (500 M rows, IVF65536, batch 1024, nprobe 32 and
256), k 10, sequential labels.  Selectors: (a) every query its own 100 "documents" of 100 consecutive labels; (b) every query its own
1 % random label set (C4: 64 distinct 1 % sets assigned round-robin -- 1024 distinct ones, 5 M labels each, would not fit beside the
48 GB of codes); (c) half the queries unfiltered, the rest as (a); (d) one 1 % set shared by every query, as a per-query filter and as
one make_filter mask.  Prints one JSON document (written to DIR when --out is given).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.bench_filter import K, SPECS, card, timed  # noqa: E402


def random_labels(N, pct, seed):
    """A pct % random subset of 0 .. N-1 (sorted): geometric gaps, so a C4-sized set takes a fraction of a second."""
    rng = np.random.default_rng(seed)
    p = pct / 100.0
    m = int(N * p * 1.05) + 64
    lab = np.cumsum(rng.geometric(p, m)) - 1
    while lab[-1] < N:
        lab = np.concatenate([lab, lab[-1] + np.cumsum(rng.geometric(p, m))])
    return lab[lab < N].astype(np.int64)


def docs(N, B, seed):
    """(a): per query, 100 random documents of 100 consecutive labels."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(B):
        starts = rng.choice(N // 100, 100, replace=False) * 100
        out.append((starts[:, None] + np.arange(100)).ravel().astype(np.int64))
    return out


def selectors(name, N, B):
    """name -> (sels, assign)."""
    a = docs(N, B, 11)
    if name == "C2":
        b = ([random_labels(N, 1, 100 + i) for i in range(B)], np.arange(B))
    else:
        b = ([random_labels(N, 1, 100 + i) for i in range(64)], np.arange(B) % 64)
    half = np.where(np.arange(B) % 2 == 0, np.arange(B), -1)
    return {"a_docs": (a, np.arange(B)), "b_1pct": b, "c_half_unfiltered": (a, half), "d_shared_1pct": ([random_labels(N, 1, 3)], np.zeros(B, np.int64))}


def selected_of(sel, N):
    s = np.zeros(N, np.uint8)
    s[sel] = 1
    return s


def blocks_read(ix, lens, qf, assign, n):
    """Selected blocks the scan read over the probed blocks of the last batch (every block for an unfiltered query)."""
    nb = (lens + 31) // 32
    probes = ix.last_probes(n)
    per_sel = {}
    read = probed = 0
    for i in range(n):
        p = probes[i][probes[i] >= 0]
        probed += int(nb[p].sum())
        s = int(assign[i])
        if s < 0:
            read += int(nb[p].sum())
            continue
        if s not in per_sel:
            off = qf.csr(s)[0].astype(np.int64)
            per_sel[s] = np.diff(off)
        read += int(per_sel[s][p].sum())
    return read / max(probed, 1)


def run(name, W, Kst, oracle, loop_q):
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
    res = {"workload": f"{name}: {N} rows, IVF{nlist}, batch {B}, k {K}", "device_bytes": ix.device_bytes, "cases": {}}
    for cname, (sels, assign) in selectors(name, N, B).items():
        c = {"selectors": len(sels), "labels_per_selector": int(np.mean([len(s) for s in sels]))}
        dsel = sels                                 # both builds take host label arrays (one copy to the device each)
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            qf = ix.make_query_filters(dsel, assign)
            c["build_ms"] = (time.perf_counter() - t0) * 1e3
        except RuntimeError as e:
            c["error"] = str(e)
            res["cases"][cname] = c
            continue
        c["bytes"] = qf.nbytes
        c["rows_per_selector"] = float(np.mean([qf.rows(i) for i in range(len(sels))]))
        torch.cuda.synchronize()                    # the sum of make_filter over the same selectors (one mask alive at a time)
        t0 = time.perf_counter()
        for s in dsel:
            f = ix.make_filter(s)
            del f
        torch.cuda.synchronize()
        c["sum_make_filter_ms"] = (time.perf_counter() - t0) * 1e3
        c["mask_bytes_each"] = 4 * int(((lens + 31) // 32).sum())
        shared = None
        if cname == "d_shared_1pct":
            shared = ix.make_filter(dsel[0])
        for nprobe in sp["nprobes"]:
            ix.nprobe = nprobe
            r = {}
            ms0, _ = timed(ix, Q, W, Kst, None)
            r["unfiltered_qps"] = B * Kst / (ms0 / 1e3)
            qfs = qf                                # the same selectors serve every timed batch
            ms, (D, I) = timed(ix, Q, W, Kst, qfs)
            r["qps"] = B * Kst / (ms / 1e3)
            r["blocks_read_share"] = blocks_read(ix, lens, qfs, assign, B)
            ix.set_profile(True)
            ix.search(Q[W + Kst - 1], K, filter=qfs)
            torch.cuda.synchronize()
            r["scan_kernel_ms"] = ix.last_scan_ms()
            ix.set_profile(False)
            if shared is not None:
                msm, (Dm, Im) = timed(ix, Q, W, Kst, shared)
                r["make_filter_qps"] = B * Kst / (msm / 1e3)
                ix.set_profile(True)
                ix.search(Q[W + Kst - 1], K, filter=shared)
                torch.cuda.synchronize()
                r["make_filter_scan_kernel_ms"] = ix.last_scan_ms()
                ix.set_profile(False)
                r["same_as_make_filter"] = bool(torch.equal(D.view(torch.int32), Dm.view(torch.int32)) and torch.equal(I, Im))
            # 16 sampled queries of the last batch against the oracle, each with its own selection
            D, I = D.cpu().numpy(), I.cpu().numpy()
            xq = Qh[W + Kst - 1].numpy()
            pick = np.linspace(0, B - 1, 16).astype(int)
            rr = ref.with_resident_lists(np.unique(ref.coarse(ref.rotate(xq[pick]), nprobe)[1]))
            ok = True
            for i in pick:
                sel = np.ones(N, np.uint8) if assign[i] < 0 else selected_of(sels[assign[i]], N)
                Dr, Ir, _ = FR.search(rr, xq[i:i + 1], K, nprobe, sel)
                ok &= bool(np.array_equal(D[i:i + 1].view(np.int32), Dr.view(np.int32)) and np.array_equal(I[i:i + 1], Ir))
            r["oracle_16_bit_identical"] = ok
            # the loop baseline over the first loop_q queries of the last batch: one-query searches with each query's mask
            nq = min(loop_q, B)
            xs = [Q[W + Kst - 1][i:i + 1].contiguous() for i in range(nq)]
            masks = [None if assign[i] < 0 else dsel[assign[i]] for i in range(nq)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(nq):
                ix.search(xs[i], K, filter=None if masks[i] is None else ix.make_filter(masks[i]))
            torch.cuda.synchronize()
            r["loop_built_in_loop_qps"] = nq / (time.perf_counter() - t0)
            if c["mask_bytes_each"] * nq <= (8 << 30):
                pre = [None if m is None else ix.make_filter(m) for m in masks]
                for i in range(min(nq, 3)):
                    ix.search(xs[i], K, filter=pre[i])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(nq):
                    ix.search(xs[i], K, filter=pre[i])
                torch.cuda.synchronize()
                r["loop_prebuilt_qps"] = nq / (time.perf_counter() - t0)
                del pre
            else:
                r["loop_prebuilt_qps"] = "not measured: the masks do not fit"
            r["loop_queries"] = nq
            c[f"nprobe{nprobe}"] = r
            del qfs
        res["cases"][cname] = c
        del qf, dsel, shared
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["C2", "C4"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loop-queries", type=int, default=64, help="queries timed in the one-query loop baseline")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_query_filters: needs a GPU")
    from oracle import ivfpq_ref as oracle
    oracle.build()
    bench.oracle_threads(oracle)
    out = {"gpu": card(), "steps": args.steps, "warmup": args.warmup, "results": {}}
    for name in args.workloads:
        out["results"][name] = run(name, args.warmup, args.steps, oracle, args.loop_queries)
        torch.cuda.empty_cache()
        print(json.dumps({name: out["results"][name]}), flush=True)
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_query_filters.json"), "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
