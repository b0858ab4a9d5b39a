"""One rank of BASELINE.json configs[3] (C4): 1B phrases, IVF65536,PQ96, 8 list-range shards, batch 1024 -- measured on ONE GPU
by building shard 0 only (125M phrases, 12 GB) and timing the rank-local work of a sharded search with the protocol the product
picks for the shape (densephrases_b200.sharded.use_query_split):
    query-split (C4):  coarse_split (this rank's 128 queries over all 65536 centroids)  +  search_assigned (LUT, plan, scan, merge)
    list-split  (C5):  coarse_local (all queries over this shard's centroids)           +  search_preassigned
(the two NCCL all-gathers, ~2 x 20 us, are not included).  Projected 8-GPU QPS = batch / rank step time.
python tools/bench_shard.py [c4|c5] [auto|single|pair|quad] [nprobe ...]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import bench
from densephrases_b200 import IvfPqIndex
from densephrases_b200.sharded import shard_ranges, use_query_split

CONFIGS = {"c4": (1_000_000_000, 65536, 8, 1024, 10),       # BASELINE.json configs[3]
           "c5": (580_000_000, 1_048_576, 8, 128, 10)}       # configs[4]: multi_wiki-scale dump, IVF1048576, eval batch 64 questions = 128 vectors
cfg = "c4"
if len(sys.argv) > 1 and sys.argv[1] in CONFIGS:
    cfg = sys.argv.pop(1)
N, NLIST, WORLD, B, K = CONFIGS[cfg]
lens = bench.uniform_lens(N, NLIST)
lo, hi = shard_ranges(lens, WORLD)[0]
ix = IvfPqIndex(NLIST)
ix.set_opq(bench.opq_matrix(1234)); ix.gen_centroids(1234); ix.gen_pq(1234); ix.set_shard(lo, hi); ix.set_lists_synthetic(lens, 1234)
torch.cuda.synchronize()
print(f"config {cfg}: N={N} nlist={NLIST} batch={B}")
print(f"shard 0: lists [{lo},{hi}), {ix.ntotal_local/1e6:.1f} M phrases, {ix.device_bytes/1e9:.1f} GB on device", flush=True)
g = torch.Generator(device="cuda").manual_seed(4321)
X = [0.5 * torch.randn((B, 768), generator=g, device="cuda") for _ in range(6)]
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
MODES = {"auto": 0, "single": 3, "pair": 2, "quad": 4}
mode = "auto"
if len(sys.argv) > 1 and sys.argv[1] in MODES:
    mode = sys.argv.pop(1)
ix.set_scan_mode(MODES[mode])
for nprobe in [int(a) for a in sys.argv[1:]] or [256, 32]:
    ix.nprobe = nprobe
    res = {}
    qsplit = use_query_split(B, WORLD, NLIST)
    per = (B + WORLD - 1) // WORLD
    recs = [torch.cat([ix.coarse_split(x[r * per:(r + 1) * per].contiguous()) for r in range(WORLD)]).contiguous() for x in X] if qsplit else None
    for name in ("coarse_local", "preassigned"):
        keys_all = []
        for x in X:      # global probes of each batch via the replicated path, re-expressed as gathered keys in slot 0
            ix.search_partial(x, K)
            pr = torch.from_numpy(ix.last_probes(B).astype(np.int64)).cuda()
            cd = torch.from_numpy(ix.last_coarse(B)).cuda()
            bits = cd.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
            fkey = torch.where(bits >= 0x80000000, (~bits) & 0xFFFFFFFF, bits | 0x80000000)
            key = (fkey << 32) | (0xFFFFFFFF - pr)
            kg = torch.zeros((WORLD, B, nprobe), dtype=torch.int64, device="cuda"); kg[0] = key
            keys_all.append(kg)
        if qsplit:
            fn = (lambda i: ix.coarse_split(X[i][:per])) if name == "coarse_local" else (lambda i: (ix.coarse_split(X[i][:per]), ix.search_assigned(recs[i], K)))
        else:
            fn = (lambda i: ix.coarse_local(X[i])) if name == "coarse_local" else (lambda i: (ix.coarse_local(X[i]), ix.search_preassigned(keys_all[i], K)))
        for i in range(3): fn(i)
        torch.cuda.synchronize(); e0.record()
        for i in range(3, 6): fn(i)
        for i in range(3, 6): fn(i)
        e1.record(); torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) / 6
    pr = ix.last_probes(B).astype(np.int64); m = (pr >= lo) & (pr < hi)
    gb = float(lens[pr[m]].sum()) * 96 / 1e9
    step = res["preassigned"]
    print(f"nprobe={nprobe} mode={mode} {'query-split' if qsplit else 'list-split'}: rank step {step:.3f} ms (before the exchange {res['coarse_local']:.3f} ms), queries/gather={ix.last_group_size()}, "
          f"algorithmic {gb:.2f} GB/rank/step = {gb/step*1000:.0f} GB/s; projected 8-GPU {B/step*1000:.0f} QPS "
          f"(HBM roofline {8*6590.9/(gb*8/B):.0f} QPS)", flush=True)
