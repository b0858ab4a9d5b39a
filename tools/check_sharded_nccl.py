"""Both sharded-search protocols on real NCCL ranks against the unsharded search of the same index (bit-identical D and I), before
after every rank adds the same batch (ShardedIvfPq.add_with_ids) and after every rank removes the same labels (ShardedIvfPq.remove_ids):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 tools/check_sharded_nccl.py
The index is synthetic (seeded, generated on the GPUs); rank 0 also builds the WHOLE index on its GPU as the reference."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, torch.distributed as dist
import bench
from densephrases_b200 import IvfPqIndex
from densephrases_b200.sharded import ShardedIvfPq

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
N, NLIST, K = 40_000_000, 4096, 10
lens = bench.uniform_lens(N, NLIST)
sh = ShardedIvfPq(NLIST, rank=rank, world=world, device=local).build_synthetic(bench.opq_matrix(7), lens, 7)
g = torch.Generator(device="cuda").manual_seed(99)
ok = True
for n, nprobe in ((1024, 64), (515, 32), (64, 256), (96, 16)):          # 515: ragged slices (the last rank's slice is padded)
    x = 0.5 * torch.randn((n, 768), generator=g, device="cuda")
    dist.broadcast(x, 0)
    sh.nprobe = nprobe
    res = {}
    for qs in (False, True):
        sh.query_split = qs
        D, I = sh.search_device(x, K)
        res[qs] = (D.clone(), I.clone())
    same = torch.equal(res[False][0], res[True][0]) and torch.equal(res[False][1], res[True][1])
    if rank == 0:
        full = IvfPqIndex(NLIST, device=local)
        full.set_opq(bench.opq_matrix(7)); full.gen_centroids(7); full.gen_pq(7); full.set_lists_synthetic(lens, 7)
        full.nprobe = nprobe
        Df, If = full.search(x, K)
        ref_ok = torch.equal(Df, res[True][0]) and torch.equal(If, res[True][1])
        del full
        torch.cuda.empty_cache()
        print(f"n={n} nprobe={nprobe} world={world}: query-split == list-split: {same}; == unsharded index: {ref_ok}", flush=True)
        ok = ok and same and ref_ok
    dist.barrier()
# growing the sharded index: every rank adds the same batch (no exchange), then both protocols == the unsharded index after the same add
xa = 0.5 * torch.randn((50_000, 768), generator=g, device="cuda")
dist.broadcast(xa, 0)
sh.add_with_ids(xa)
x = 0.5 * torch.randn((1024, 768), generator=g, device="cuda")
dist.broadcast(x, 0)
sh.nprobe = 64
res = {}
for qs in (False, True):
    sh.query_split = qs
    res[qs] = tuple(t.clone() for t in sh.search_device(x, K))
if rank == 0:
    full = IvfPqIndex(NLIST, device=local)
    full.set_opq(bench.opq_matrix(7)); full.gen_centroids(7); full.gen_pq(7); full.set_lists_synthetic(lens, 7)
    full.add(xa)
    full.nprobe = 64
    Df, If = full.search(x, K)
    add_ok = all(torch.equal(Df, res[qs][0]) and torch.equal(If, res[qs][1]) for qs in (False, True)) and full.ntotal == sh.ntotal
    print(f"after add of {xa.shape[0]} vectors, world={world}: both protocols == unsharded grown index: {add_ok}", flush=True)
    ok = ok and add_ok
dist.barrier()
# shrinking it: every rank removes the same label range and label set (per-list counts all-reduced, list lengths synchronised), then
# both protocols == the unsharded index after the same removes
sel_set = torch.randint(0, N + xa.shape[0], (20_000,), generator=g, device="cuda")
dist.broadcast(sel_set, 0)
sels = (range(N // 3, N // 3 + 1_000_000), sel_set.cpu().numpy())
n_rm = [sh.remove_ids(s) for s in sels]
res = {}
for qs in (False, True):
    sh.query_split = qs
    res[qs] = tuple(t.clone() for t in sh.search_device(x, K))
if rank == 0:
    full = IvfPqIndex(NLIST, device=local)
    full.set_opq(bench.opq_matrix(7)); full.gen_centroids(7); full.gen_pq(7); full.set_lists_synthetic(lens, 7)
    full.add(xa)
    n_full = [full.remove_ids(s) for s in sels]
    full.nprobe = 64
    Df, If = full.search(x, K)
    rm_ok = all(torch.equal(Df, res[qs][0]) and torch.equal(If, res[qs][1]) for qs in (False, True)) and full.ntotal == sh.ntotal \
        and n_full == n_rm
    print(f"after removing {sum(n_rm)} rows, world={world}: both protocols == unsharded index after the same removes: {rm_ok}", flush=True)
    ok = ok and rm_ok
dist.barrier()
if rank == 0:
    print("SHARDED NCCL CHECK", "PASSED" if ok else "FAILED", flush=True)
dist.destroy_process_group()
