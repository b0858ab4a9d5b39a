"""Growing a resident index (dph_index_add_with_ids) on one GPU: start from a trained, empty OPQ96 / IVF{nlist} / PQ96 index
(synthetic centroids and codebooks) and add near-vectors (rotated image = a random centroid + noise) from device buffers in chunks.
Reports end-to-end vectors/s (profiling off), the per-stage CUDA-event times of a second, profiled pass (rotation, coarse, PQ encode,
re-layout + scatter), the PQ-encode kernel against the FP32 peak and the re-layout's bytes against HBM bandwidth, and two baselines:
build_index.add_to_index (PyTorch, same GPU, TF32 off) and the oracle's ref_encode on the host cores.
    python tools/bench_add.py [--nlist 4096 65536] [--total 10000000] [--chunk 1000000] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

FP32_PEAK, HBM_PEAK = 67e12, 3.35e12          # H100 SXM data sheet (dense FP32, HBM3)
SEED = 5


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def model(nlist):
    from oracle import ivfpq_ref as R
    A = np.linalg.qr(np.random.default_rng(SEED).standard_normal((768, 768)))[0].astype(np.float32)
    return A, R.gen_centroids(SEED, 0, nlist), R.gen_pq(SEED)


def near_batch(A_t, C_t, n, g):
    lists = torch.randint(0, C_t.shape[0], (n,), generator=g, device="cuda")
    return ((C_t[lists] + 0.3 * torch.randn((n, 768), generator=g, device="cuda")) @ A_t).contiguous()


def grow(nlist, total, chunk, profile):
    from densephrases_b200 import IvfPqIndex
    A, Cm, _ = model(nlist)
    ix = IvfPqIndex(nlist)
    ix.set_opq(A); ix.gen_centroids(SEED); ix.gen_pq(SEED)
    ix.set_lists(np.zeros(nlist, np.int64), np.zeros((0, 96), np.uint8))
    ix.set_profile(profile)
    A_t, C_t = torch.from_numpy(A).cuda(), torch.from_numpy(Cm).cuda()
    g = torch.Generator(device="cuda").manual_seed(SEED)
    warm = near_batch(A_t, C_t, 4096, g)
    ix.encode(warm)                                           # module load, coarse-path set-up (centroid split)
    scratch = IvfPqIndex(nlist)                               # the re-layout and sort kernels, on a throwaway index
    scratch.set_opq(A); scratch.gen_centroids(SEED); scratch.gen_pq(SEED)
    scratch.set_lists(np.zeros(nlist, np.int64), np.zeros((0, 96), np.uint8))
    scratch.add(warm); scratch.add(warm)
    del scratch
    secs, stages, relayout_bytes = 0.0, np.zeros(4), 0.0
    for o in range(0, total, chunk):
        x = near_batch(A_t, C_t, min(chunk, total - o), g)
        old = ix.ntotal
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.add(x)                                             # synchronises the stream before it returns
        secs += time.perf_counter() - t0
        if profile:
            stages += ix.last_add_ms()
        # bytes the re-layout + scatter must move (rows, padding not counted; the sorts not counted): old codes + labels read and
        # written, old direct-map pairs read and written, the batch's codes + labels read and its direct-map pairs written
        added = ix.ntotal - old
        relayout_bytes += old * (2 * 104 + 2 * 16) + added * (104 + 104 + 16)
        del x
    out = {"nlist": nlist, "vectors": total, "chunk": chunk, "seconds": secs, "vectors_per_s": total / secs, "device_bytes": ix.device_bytes}
    if profile:
        enc_flop = total * 96 * 256 * 8 * 3                   # per (vector, m, j, t): one FSUB + one FFMA (2 flops)
        out.update(stage_ms=dict(zip(("rotation", "coarse", "pq_encode", "relayout_scatter"), stages.round(2).tolist())),
                   pq_encode_tflops=enc_flop / (stages[2] / 1e3) / 1e12, pq_encode_frac_fp32_peak=enc_flop / (stages[2] / 1e3) / FP32_PEAK,
                   relayout_gbytes=relayout_bytes / 1e9, relayout_frac_hbm_peak=relayout_bytes / (stages[3] / 1e3) / HBM_PEAK)
    return out


def torch_baseline(nlist, n):
    from densephrases_b200.build_index import add_to_index
    torch.backends.cuda.matmul.allow_tf32 = False
    A, Cm, pq = model(nlist)
    x = near_batch(torch.from_numpy(A).cuda(), torch.from_numpy(Cm).cuda(), n, torch.Generator(device="cuda").manual_seed(1)).cpu().numpy()
    add_to_index(A, Cm, pq, x[:4096], device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    add_to_index(A, Cm, pq, x, device="cuda")
    torch.cuda.synchronize()
    return {"vectors": n, "vectors_per_s": n / (time.perf_counter() - t0)}


def oracle_baseline(nlist, n):
    from oracle import encode_ref as E
    A, Cm, pq = model(nlist)
    x = ((Cm[np.random.default_rng(2).integers(0, nlist, n)] + 0.3 * np.random.default_rng(3).standard_normal((n, 768))) @ A).astype(np.float32)
    t0 = time.perf_counter()
    E.encode(A, Cm, pq, x)
    return {"vectors": n, "vectors_per_s": n / (time.perf_counter() - t0), "threads": E.lib().ref_num_threads(), "nproc": os.cpu_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nlist", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--total", type=int, default=10_000_000)
    ap.add_argument("--chunk", type=int, default=1_000_000)
    ap.add_argument("--baseline-n", type=int, default=200_000)
    ap.add_argument("--oracle-n", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_add needs a GPU")
    from oracle import encode_ref, ivfpq_ref
    ivfpq_ref.build()
    encode_ref.build()
    info = gpu_info()
    rows = []
    for nlist in a.nlist:
        r = grow(nlist, a.total, a.chunk, profile=False)
        r["profiled"] = grow(nlist, a.total, a.chunk, profile=True)
        r["torch_add_to_index"] = torch_baseline(nlist, a.baseline_n)
        r["oracle_ref_encode"] = oracle_baseline(nlist, max(100, a.oracle_n * 4096 // nlist))      # same host time per workload
        r.update(info)
        rows.append(r)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    print(f"\n{info}")
    print(f"{'nlist':>7} {'vec/s':>10} {'rot ms':>8} {'coarse ms':>10} {'pq ms':>8} {'relayout ms':>11} {'pq %fp32':>9} {'relayout %hbm':>13} "
          f"{'torch vec/s':>11} {'oracle vec/s':>12}")
    for r in rows:
        p = r["profiled"]; s = p["stage_ms"]
        print(f"{r['nlist']:>7} {r['vectors_per_s']:>10.0f} {s['rotation']:>8.1f} {s['coarse']:>10.1f} {s['pq_encode']:>8.1f} {s['relayout_scatter']:>11.1f} "
              f"{100 * p['pq_encode_frac_fp32_peak']:>8.1f}% {100 * p['relayout_frac_hbm_peak']:>12.1f}% {r['torch_add_to_index']['vectors_per_s']:>11.0f} "
              f"{r['oracle_ref_encode']['vectors_per_s']:>12.0f}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_add.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
