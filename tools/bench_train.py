"""Training a phrase index on one GPU (IvfPqIndex.train: OPQ, spherical k-means coarse quantizer, residual PQ; DESIGN.md 3.3) on
synthetic clustered vectors generated on the GPU from a seed.  Per workload: the median of 3 unprofiled passes of every stage, the
CUDA-event stage times of one profiled pass (assign, sort + update, split + renorm), the assignment's FP32 rate against the data-sheet
peaks and the update's bytes against HBM bandwidth, and recall@10 of the trained index (filled with the training rows) on held-out
queries against exact MIPS.  At IVF4096 the torch trainer (build_index.train_index, TF32 off) is timed and scored on the same data;
at IVF65536 its n x nlist score matrix is reported by arithmetic.  Each run first checks a small training bit for bit against the
oracle.
    python tools/bench_train.py [--workloads 4096:1048576 65536:2555904] [--passes 3] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

FP32_PEAK, TF32_PEAK, HBM_PEAK = 67e12, 495e12, 3.35e12     # H100 SXM data sheet (dense FP32, dense TF32, HBM3)
SEED = 7


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def clustered(n, seed, groups=20000, spread=0.6):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn((groups, 768), generator=g, device="cuda")
    a = torch.randint(0, groups, (n,), generator=g, device="cuda")
    x = centres[a]
    x.add_(spread * torch.randn((n, 768), generator=g, device="cuda"))
    return x.contiguous(), centres


def check_oracle():
    from densephrases_b200 import IvfPqIndex
    from oracle import train_ref as T
    A = np.linalg.qr(np.random.default_rng(SEED).standard_normal((768, 768)))[0].astype(np.float32)
    x = clustered(4096, 3, groups=64)[0].cpu().numpy() @ A
    x = np.ascontiguousarray(x, dtype=np.float32)
    ix = IvfPqIndex(256)
    ix.set_opq(A)
    obj, _ = ix.train_coarse(x, niter=2, seed=SEED)
    Cr, objr, _ = T.train_coarse(x, A, 256, 2, SEED)
    ix.train_pq(x, niter=2, seed=SEED)
    ok = (np.array_equal(ix.centroids().view(np.int32), Cr.view(np.int32)) and np.array_equal(obj, objr)
          and np.array_equal(ix.pq_codebooks().view(np.int32), T.train_pq(x, A, Cr, 2, SEED).view(np.int32)))
    assert ok, "training differs from the oracle"
    return ok


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def recall_at_10(ix, x, q, exact, nprobe=64):
    ix.set_lists(np.zeros(ix.nlist, np.int64), np.zeros((0, 96), np.uint8))          # trained, empty
    ix.add_with_ids(x, None)
    ix.nprobe = nprobe
    I = ix.search(q, 10)[1].cpu().numpy()
    return float(np.mean([len(set(I[i]) & set(exact[i])) / 10 for i in range(len(q))]))


def workload(nlist, n, passes, torch_baseline):
    from densephrases_b200 import IvfPqIndex
    x, centres = clustered(n, SEED)
    g = torch.Generator(device="cuda").manual_seed(SEED + 1)
    q = (centres[torch.randint(0, len(centres), (1000,), generator=g, device="cuda")]
         + 0.6 * torch.randn((1000, 768), generator=g, device="cuda")).contiguous()
    torch.backends.cuda.matmul.allow_tf32 = False
    exact = torch.topk(q @ x.T, 10, dim=1).indices.cpu().numpy()
    res = {"nlist": nlist, "n": n, "rows_per_centroid": n / nlist}
    stages = {"opq": [], "coarse": [], "pq": []}
    ix = None
    for p in range(passes + 1):
        prof = p == passes                                         # last pass: profiled, for the stage split
        ix = IvfPqIndex(nlist)
        ix.set_profile(prof)
        t_opq, _ = timed(lambda: ix.train_opq(x, niter=10, seed=SEED))
        t_c, (obj, nsplit) = timed(lambda: ix.train_coarse(x, niter=10, seed=SEED))
        cms = ix.last_train_ms().astype(np.float64) if prof else None
        t_pq, _ = timed(lambda: ix.train_pq(x, niter=25, seed=SEED))
        pms = ix.last_train_ms().astype(np.float64) if prof else None
        if not prof:
            stages["opq"].append(t_opq); stages["coarse"].append(t_c); stages["pq"].append(t_pq)
    med = {k: float(np.median(v)) for k, v in stages.items()}
    res["median_s"] = dict(med, total=sum(med.values()))
    res["coarse_profiled_ms"] = dict(zip(["assign", "sort_update", "split_renorm"], cms.round(2).tolist()))
    res["pq_profiled_ms"] = dict(zip(["assign", "sort_update", "split"], pms.round(2).tolist()))
    ns = min(n, 256 * nlist)
    flops = 2.0 * ns * nlist * 768 * 10                            # 10 assignment passes of the coarse quantizer
    res["coarse_assign_tflops"] = flops / (cms[0] / 1e3) / 1e12
    res["coarse_assign_vs_fp32_peak"] = res["coarse_assign_tflops"] * 1e12 / FP32_PEAK
    res["coarse_assign_vs_tf32_peak"] = res["coarse_assign_tflops"] * 1e12 / TF32_PEAK
    upd_bytes = 10 * ns * 768 * 4.0                                # every update reads the sample once
    res["coarse_update_GBps"] = upd_bytes / (cms[1] / 1e3) / 1e9
    res["coarse_update_vs_hbm"] = upd_bytes / (cms[1] / 1e3) / HBM_PEAK
    res["coarse_obj_first_last"] = [float(obj[0]), float(obj[-1])]
    res["coarse_nsplit"] = int(nsplit.sum())
    res["gpu_recall_at_10"] = recall_at_10(ix, x, q, exact)
    if torch_baseline:
        from densephrases_b200.build_index import train_index
        xn = x.cpu().numpy()
        t_t, (A, Cm, pq) = timed(lambda: train_index(xn, nlist, niter_opq=10, niter_km=10, niter_pq=25, seed=SEED, device="cuda"))
        res["torch_train_s"] = t_t
        tix = IvfPqIndex(nlist)
        tix.set_opq(A); tix.set_centroids(Cm); tix.set_pq(pq)
        res["torch_recall_at_10"] = recall_at_10(tix, x, q, exact)
    else:
        score_bytes = 39 * nlist * nlist * 4.0                     # train_index's n x nlist fp32 matrix at faiss' 39 rows per centroid
        res["torch_train"] = f"not run: its score matrix alone is {score_bytes / 1e9:.0f} GB at 39 rows per centroid"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["4096:1048576", "65536:2555904"])
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"info": gpu_info(), "oracle_check": check_oracle(), "workloads": []}
    for w in a.workloads:
        nlist, n = (int(v) for v in w.split(":"))
        out["workloads"].append(workload(nlist, n, a.passes, torch_baseline=(nlist <= 4096 and not a.no_torch)))
        print(json.dumps(out["workloads"][-1], default=float), flush=True)
    print(json.dumps(out, default=float))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_train.json"), "w") as f:
            json.dump(out, f, indent=1, default=float)


if __name__ == "__main__":
    main()
