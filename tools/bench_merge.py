"""Merging indexes (dph_index_merge_from) on one GPU: synthetic OPQ96 / IVF{nlist} / PQ96 indexes (synthetic centroids, codebooks and
codes, sequential labels), the sources sharing the destination's tables, merged with add_id = the destination's ntotal (the offsets of
the reference's sub-index jobs).  Two workloads:
  c2      one 10 M-row source into a 100 M-row IVF4096 index (the C2 shape of bench.py)
  ivf64k  four 10 M-row sources at once into an IVF65536 index of --big rows (default 400 M)
Each pass starts from a freshly built destination (the merge turns its sequential labels into explicit ones).  Reports the end-to-end
time of the synchronous call (median and range of --passes unprofiled passes), the stage times of one more, profiled pass (plan +
alloc, block moves, source rows, direct map), the bytes the merge must read and write against 3.35 TB/s, device_bytes, and the card
and power limit read in the same run.  A destination too large for the old and the new buffers at once is rejected by the merge with
the index unchanged; that is reported as such.
    python tools/bench_merge.py [--workloads c2 ivf64k] [--big 400000000] [--passes 3] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

HBM_PEAK = 3.35e12          # H100 SXM data sheet (HBM3)
SEED = 5


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def lengths(nlist, n, seed):
    rng = np.random.default_rng(seed)
    w = np.exp(rng.normal(0, 0.5, nlist))
    return rng.multinomial(n, w / w.sum()).astype(np.int64)


def synthetic(nlist, lens, code_seed):
    from densephrases_b200 import IvfPqIndex
    A = np.linalg.qr(np.random.default_rng(SEED).standard_normal((768, 768)))[0].astype(np.float32)
    ix = IvfPqIndex(nlist)
    ix.set_opq(A); ix.gen_centroids(SEED); ix.gen_pq(SEED)
    ix.set_lists_synthetic(lens, code_seed)
    return ix


def merge_bytes(n_dest, n_src):
    """What the merge must read and write, padding not counted: the destination's codes read and written, its labels written (they
    were sequential), each source row's code and label read and written, one direct-map pair (16 B) written per row."""
    return n_dest * (2 * 96 + 8) + n_src * 2 * (96 + 8) + (n_dest + n_src) * 16


def run(name, nlist, n_dest, n_src, k_src, passes):
    srcs = [synthetic(nlist, lengths(nlist, n_src, 100 + s), 100 + s) for s in range(k_src)]
    lens = lengths(nlist, n_dest, 1)
    out = {"workload": name, "nlist": nlist, "dest_rows": n_dest, "sources": k_src, "source_rows": n_src}
    secs, stages = [], None
    for p in range(passes + 1):
        ix = synthetic(nlist, lens, 1)
        profile = p == passes
        ix.set_profile(profile)
        b0 = ix.device_bytes
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        try:
            ix.merge_from(srcs, add_id=n_dest)
        except RuntimeError as e:
            out.update(rejected=str(e), unchanged=bool(ix.ntotal == n_dest and ix.device_bytes == b0), device_bytes_before=b0)
            return out
        t = time.perf_counter() - t0
        assert ix.ntotal == n_dest + k_src * n_src
        if profile:
            stages = ix.last_merge_ms()
            out["device_bytes"] = ix.device_bytes
        else:
            secs.append(t)
        del ix
        torch.cuda.empty_cache()
    mb = merge_bytes(n_dest, k_src * n_src)
    med = float(np.median(secs))
    out.update(seconds_median=med, seconds_min=min(secs), seconds_max=max(secs),
               stage_ms=dict(zip(("plan_alloc", "block_moves", "source_rows", "direct_map"), stages.round(2).tolist())),
               gbytes=mb / 1e9, frac_hbm_peak_e2e=mb / med / HBM_PEAK,
               frac_hbm_peak_device=mb / (float(stages[1:].sum()) / 1e3) / HBM_PEAK)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["c2", "ivf64k"])
    ap.add_argument("--big", type=int, nargs="+", default=[400_000_000], help="destination rows of the ivf64k workload (tried in turn)")
    ap.add_argument("--source-rows", type=int, default=10_000_000)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_merge needs a GPU")
    info = gpu_info()
    rows = []
    for w in a.workloads:
        specs = [("c2", 4096, 100_000_000, 1)] if w == "c2" else [("ivf64k", 65536, n, 4) for n in a.big]
        for name, nlist, n_dest, k in specs:
            r = run(name, nlist, n_dest, a.source_rows, k, a.passes)
            r.update(info)
            rows.append(r)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()
    print(f"\n{info}")
    print(f"{'workload':>8} {'dest rows':>11} {'sources':>7} {'median s':>9} {'min-max s':>13} {'plan ms':>8} {'blocks ms':>9} {'rows ms':>8} "
          f"{'dmap ms':>8} {'GB':>6} {'e2e %hbm':>8} {'dev %hbm':>8}")
    for r in rows:
        if "rejected" in r:
            print(f"{r['workload']:>8} {r['dest_rows']:>11} {r['sources']:>7}  rejected (index unchanged: {r['unchanged']}): {r['rejected'][:90]}")
            continue
        s = r["stage_ms"]
        print(f"{r['workload']:>8} {r['dest_rows']:>11} {r['sources']:>7} {r['seconds_median']:>9.3f} {r['seconds_min']:>6.3f}-{r['seconds_max']:<6.3f} "
              f"{s['plan_alloc']:>8.1f} {s['block_moves']:>9.1f} {s['source_rows']:>8.1f} {s['direct_map']:>8.1f} {r['gbytes']:>6.1f} "
              f"{100 * r['frac_hbm_peak_e2e']:>7.1f}% {100 * r['frac_hbm_peak_device']:>7.1f}%")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_merge.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
