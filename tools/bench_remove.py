"""Removing vectors from a resident index (dph_index_remove_ids) on one GPU.
Workloads:
  - the 10 M-vector OPQ96 / IVF65536 / PQ96 index tools/bench_add.py builds (near-vectors added in 1 M chunks, labels 0 .. 10 M - 1),
    in turn: one document (100 consecutive labels), 1 % of the labels at random, a 1 M-label range;
  - a 400 M-row synthetic IVF65536 index (38 GB of codes, more than half the device) with sequential labels: a 1 M-label range (the
    first remove also makes the labels explicit, +24 B per row), then a second 1 M-label range.
Reports the end-to-end time (median, min and max over --reps unprofiled passes, each from the same starting index), the CUDA-event stage
times of one more, profiled pass (mark + plan, row moves + block shift, direct map), the bytes the hole fills and
the block shift must move (read + write) and the direct-map bytes, each against the HBM3 data-sheet bandwidth, the largest temporary
allocation, and the host oracle's time (oracle/remove_ref.c, the literal faiss loop, one host core; the copies of the arrays it works on are
made before the clock starts) for the two small workloads.
    python tools/bench_remove.py [--total 10000000] [--big-rows 400000000] [--out DIR]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

from bench_add import SEED, gpu_info, model, near_batch

HBM_PEAK = 3.35e12          # H100 SXM data sheet (HBM3)


def plan_bytes(lens_old, lens_new, holes, dm_n):
    """Bytes that must move: hole fills (96 B code + 8 B label, read + write per moved row), the block shift (3072 B codes + 256 B
    labels per block, read + write, for every block after the first list whose block count dropped), the direct map (16 B per pair,
    read + write)."""
    nb_old, nb_new = (lens_old + 31) // 32, (lens_new + 31) // 32
    dropped = np.flatnonzero(nb_old != nb_new)
    shift_blocks = int(nb_new[dropped[0] + 1:].sum()) if len(dropped) else 0
    return {"hole_rows": int(holes), "shift_blocks": shift_blocks, "rows_bytes": int(holes * 104 * 2 + shift_blocks * 3328 * 2),
            "dm_bytes": int(dm_n * 16 * 2)}


def holes_from_ids(lens, ids, sel_mask):
    """Removed rows below L' of their list (the moves the closed form makes)."""
    li = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(len(ids)) - np.repeat(np.cumsum(lens) - lens, lens)
    per = np.bincount(li, weights=sel_mask, minlength=len(lens)).astype(np.int64)
    return int((sel_mask & (j < (lens - per)[li])).sum())


def timed_remove(ix, sel):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = ix.remove_ids(sel)                                    # synchronises the stream before it returns
    return n, time.perf_counter() - t0


def report(name, n, e2e_s, ms, pb, tmp_bytes, extra=None):
    """e2e_s: end-to-end seconds of the unprofiled repetitions; ms: stage times of the profiled pass."""
    ms = [float(v) for v in ms]
    e2e = np.array(e2e_s) * 1e3
    r = {"workload": name, "removed": n, "ms": float(np.median(e2e)), "ms_min": float(e2e.min()), "ms_max": float(e2e.max()),
         "reps": len(e2e), "stage_ms": dict(zip(("mark_plan", "moves_shift", "direct_map"), np.round(ms, 3).tolist())),
         "tmp_peak_bytes": tmp_bytes, **pb}
    r["moves_shift_frac_hbm"] = pb["rows_bytes"] / (ms[1] / 1e3) / HBM_PEAK if ms[1] > 0 else None
    r["direct_map_frac_hbm"] = pb["dm_bytes"] / (ms[2] / 1e3) / HBM_PEAK if ms[2] > 0 else None
    if extra:
        r.update(extra)
    print(json.dumps(r), flush=True)
    return r


def warm(nlist):
    from densephrases_b200 import IvfPqIndex
    A, _, _ = model(nlist)
    ix = IvfPqIndex(nlist)
    ix.set_opq(A); ix.gen_centroids(SEED); ix.gen_pq(SEED)
    ix.set_lists_synthetic(np.full(nlist, 40, np.int64), SEED)
    ix.remove_ids(np.arange(0, 4000, 7, dtype=np.int64))
    ix.remove_ids(range(100, 3000))


def grown_lists(nlist, total, chunk):
    """The list-major arrays of the index tools/bench_add.py grows (device state of add_with_ids == set_lists of these arrays)."""
    from densephrases_b200 import IvfPqIndex
    A, Cm, _ = model(nlist)
    ix = IvfPqIndex(nlist)
    ix.set_opq(A); ix.gen_centroids(SEED); ix.gen_pq(SEED)
    ix.set_lists(np.zeros(nlist, np.int64), np.zeros((0, 96), np.uint8))
    A_t, C_t = torch.from_numpy(A).cuda(), torch.from_numpy(Cm).cuda()
    g = torch.Generator(device="cuda").manual_seed(SEED)
    for o in range(0, total, chunk):
        ix.add(near_batch(A_t, C_t, min(chunk, total - o), g))
    return ix.lists()


def small_workloads(a, rows):
    """Each pass starts from the same grown index; a.reps unprofiled passes give the end-to-end times, one profiled pass the stages."""
    from densephrases_b200 import IvfPqIndex
    from oracle import remove_ref as RR
    nlist = 65536
    A, Cm, pq = model(nlist)
    base = grown_lists(nlist, a.total, a.chunk)
    torch.cuda.empty_cache()
    rng = np.random.default_rng(3)
    doc0 = int(rng.integers(0, a.total - 100))
    work = (("one document: 100 consecutive labels", range(doc0, doc0 + 100)),
            ("1% random labels", rng.choice(a.total, a.total // 100, replace=False).astype(np.int64)),
            ("1M-label range", range(a.total // 2, a.total // 2 + 1_000_000)))
    e2e = [[] for _ in work]
    for rep in range(a.reps + 1):
        profile = rep == a.reps
        ix = IvfPqIndex.from_arrays(A, Cm, pq, *base)
        ix.set_profile(profile)
        for w, (name, sel) in enumerate(work):
            if not profile:
                e2e[w].append(timed_remove(ix, sel)[1])
                continue
            lens, codes, ids = ix.lists()
            mask = np.isin(ids, sel) if isinstance(sel, np.ndarray) else (ids >= sel.start) & (ids < sel.stop)
            dm_n = len(ids)
            n, _ = timed_remove(ix, sel)
            pb = plan_bytes(lens, ix.list_len(), holes_from_ids(lens, ids, mask), dm_n - n)
            extra = {"index": f"IVF{nlist}, {dm_n} rows (grown by adds)"}
            if not name.startswith("1M"):         # the C loop alone, on copies made beforehand (one host core)
                per = np.zeros(nlist, np.int64)
                lens, codes, ids = lens.copy(), np.ascontiguousarray(codes), ids.copy()
                s, lo, hi = RR.selector(sel)
                t0 = time.perf_counter()
                RR.ref_remove_inplace(lens, codes, ids, s, lo, hi, per)
                extra["host_oracle_ms"] = (time.perf_counter() - t0) * 1e3
            del codes
            rows.append(report(name, n, e2e[w], ix.last_remove_ms(), pb, ix.last_remove_tmp_bytes(), extra))
        del ix
        torch.cuda.empty_cache()


def big_workload(a, rows):
    """Each pass builds the synthetic index anew: the first remove also makes its labels explicit."""
    from densephrases_b200 import IvfPqIndex
    nlist = 65536
    lens = np.full(nlist, a.big_rows // nlist, np.int64)
    lens[: a.big_rows - int(lens.sum())] += 1
    A, _, _ = model(nlist)
    work = (("1M-label range, 400M synthetic (labels become explicit)", a.big_rows // 3),
            ("1M-label range, 400M synthetic (explicit labels)", a.big_rows // 2))
    e2e = [[] for _ in work]
    for rep in range(a.reps + 1):
        profile = rep == a.reps
        ix = IvfPqIndex(nlist)
        ix.set_opq(A); ix.gen_centroids(SEED); ix.gen_pq(SEED)
        ix.set_lists_synthetic(lens, SEED)
        ix.set_profile(profile)
        b0 = ix.device_bytes
        start = np.concatenate([[0], np.cumsum(lens)])
        for w, (name, lo) in enumerate(work):
            hi = lo + 1_000_000
            if not profile:
                e2e[w].append(timed_remove(ix, range(lo, hi))[1])
                continue
            old = ix.list_len()
            dm_n = int(old.sum())
            s = np.clip(lo - start[:-1], 0, old); e = np.clip(hi - start[:-1], 0, old)       # labels are list-major rows: one interval per list
            n, _ = timed_remove(ix, range(lo, hi))
            new = ix.list_len()
            holes = int(np.maximum(0, np.minimum(e, new) - s).sum())
            pb = plan_bytes(old, new, holes, dm_n - n)
            rows.append(report(name, n, e2e[w], ix.last_remove_ms(), pb, ix.last_remove_tmp_bytes(),
                               {"index": f"IVF{nlist}, {dm_n} rows (synthetic)", "codes_gb": dm_n * 96 / 1e9, "device_bytes_before": b0,
                                "device_bytes_after": ix.device_bytes}))
            b0 = ix.device_bytes
            start = np.concatenate([[0], np.cumsum(new)])
        del ix
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--total", type=int, default=10_000_000)
    ap.add_argument("--chunk", type=int, default=1_000_000)
    ap.add_argument("--big-rows", type=int, default=400_000_000)
    ap.add_argument("--reps", type=int, default=3, help="unprofiled passes per workload (end-to-end times); one more, profiled, gives the stages")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_remove needs a GPU")
    from oracle import ivfpq_ref, remove_ref
    ivfpq_ref.build()
    remove_ref.build()
    info = gpu_info()
    print(json.dumps(info), flush=True)
    warm(1024)
    rows = []
    small_workloads(a, rows)
    if a.big_rows > 0:
        big_workload(a, rows)
    for r in rows:
        r.update(info)
    print(f"\n{info}")
    print(f"{'workload':<58} {'removed':>9} {'ms':>9} {'min-max ms':>15} {'mark+plan':>10} {'moves+shift':>12} {'dmap':>8} {'rows GB':>8} {'%hbm':>6} "
          f"{'dmap GB':>8} {'%hbm':>6} {'oracle ms':>10}")
    for r in rows:
        s = r["stage_ms"]
        f1 = r["moves_shift_frac_hbm"]; f2 = r["direct_map_frac_hbm"]
        print(f"{r['workload']:<58} {r['removed']:>9} {r['ms']:>9.2f} {r['ms_min']:>7.2f}-{r['ms_max']:<7.2f} {s['mark_plan']:>10.3f} {s['moves_shift']:>12.3f} {s['direct_map']:>8.3f} "
              f"{r['rows_bytes'] / 1e9:>8.3f} {100 * f1 if f1 else 0:>5.1f}% {r['dm_bytes'] / 1e9:>8.3f} {100 * f2 if f2 else 0:>5.1f}% "
              f"{r.get('host_oracle_ms', float('nan')):>10.1f}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_remove.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
