"""One rank of C4 (shard 0 of 8; batch 1024) at nprobe 256 and 32: the list-split against the query-split coarse quantizer, with the
time before the exchange and the scan time, and whether both give the same results:  python tools/bench_variants.py shard"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import bench
from densephrases_b200 import IvfPqIndex
from densephrases_b200.sharded import shard_ranges

ev = lambda: torch.cuda.Event(enable_timing=True)


def timeit(fn, reps, warm=3):
    for i in range(warm): fn(i)
    torch.cuda.synchronize(); e0, e1 = ev(), ev(); e0.record()
    for i in range(reps): fn(warm + i)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


N, NLIST, WORLD, B, K = 1_000_000_000, 65536, 8, 1024, 10
lens = bench.uniform_lens(N, NLIST)
lo, hi = shard_ranges(lens, WORLD)[0]
ix = IvfPqIndex(NLIST)
ix.set_opq(bench.opq_matrix(1234)); ix.gen_centroids(1234); ix.gen_pq(1234); ix.set_shard(lo, hi); ix.set_lists_synthetic(lens, 1234)
ix.set_profile(True)
g = torch.Generator(device="cuda").manual_seed(4321)
X = [0.5 * torch.randn((B, 768), generator=g, device="cuda") for _ in range(6)]
for nprobe in (256, 32):
    ix.nprobe = nprobe
    keys_all = []
    for x in X:
        ix.search_partial(x, K)
        pr = torch.from_numpy(ix.last_probes(B).astype(np.int64)).cuda()
        cd = torch.from_numpy(ix.last_coarse(B)).cuda()
        bits = cd.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
        fkey = torch.where(bits >= 0x80000000, (~bits) & 0xFFFFFFFF, bits | 0x80000000)
        kg = torch.zeros((WORLD, B, nprobe), dtype=torch.int64, device="cuda"); kg[0] = (fkey << 32) | (0xFFFFFFFF - pr)
        keys_all.append(kg)
    # records of the query-split protocol: every "rank" assigns its slice of 128 queries over all lists (here: this GPU, 8 times)
    per = B // WORLD
    recs = [torch.cat([ix.coarse_split(x[r * per:(r + 1) * per].contiguous()) for r in range(WORLD)]).contiguous() for x in X]
    base = None
    for proto in ("list-split", "query-split"):
        if proto == "list-split":
            fn = lambda i: (ix.coarse_local(X[i % 6]), ix.search_preassigned(keys_all[i % 6], K))
            pre = lambda i: ix.coarse_local(X[i % 6])
        else:
            fn = lambda i: (ix.coarse_split(X[i % 6][:per]), ix.search_assigned(recs[i % 6], K))
            pre = lambda i: ix.coarse_split(X[i % 6][:per])
        ms_pre = timeit(pre, 12, warm=3)
        ms = timeit(fn, 12, warm=3)
        scan = np.mean(ix.profile_scan_ms()[-12:])
        _, (D, I, G) = fn(0)
        if base is None: base = (D.clone(), I.clone())
        same = bool((D == base[0]).all() and (I == base[1]).all())
        print(f"C4 shard nprobe {nprobe} {proto}: rank step {ms:.3f} ms (before the exchange {ms_pre:.3f}) -> {B / ms * 1000:.0f} QPS on 8 GPUs, "
              f"scan {scan:.3f} ms, same results {same}", flush=True)
