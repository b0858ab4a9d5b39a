"""CPU: per-query filters (DESIGN.md 3.7).  The numpy restatement equals the C filtered oracle run query by query; the CSR restatement
expands to the row mask of tests/filter_ref.py; MIPS' document -> label-runs index gives the labels of the np.isin rule; both sharded
protocols over gloo (world size 2, oracle shards) with per-query selections equal the unsharded definition."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import filter_ref as FR
from tests.filter_ref import np_filtered_search, np_mask
from tests.helpers import assert_topk_equal, near_queries, opq_matrix
from tests.query_filter_ref import csr_mask, np_csr, query_filtered_search
from tests.test_filter_cpu import FilterIndexStandIn, ragged_ref, selectors, synthetic_idx2id

SEED = 37


@pytest.mark.parametrize("explicit", [True, False])
@pytest.mark.parametrize("k", [1, 10, 100])
def test_restatement_equals_the_oracle_query_by_query(oracle, explicit, k):
    ref = ragged_ref(oracle, explicit=explicit)
    x = near_queries(ref, 9, SEED)
    sels = list(selectors(ref).values())
    selected = [FR.selected_rows(ref, s) for s in sels]
    assign = np.array([0, 1, -1, 2, 3, 4, 5, 0, -1])
    for nprobe in (1, 4, 12):
        D, I = query_filtered_search(ref, x, k, nprobe, selected, assign)
        Dn, In = query_filtered_search(ref, x, k, nprobe, selected, assign, search=np_filtered_search)
        assert_topk_equal(D, I, Dn, In, f"nprobe={nprobe}")
        for i in range(len(x)):               # row i alone, with its own selection
            sel = np.ones(ref.ntotal, np.uint8) if assign[i] < 0 else selected[assign[i]]
            Di, Ii, _ = FR.search(ref, x[i:i + 1], k, nprobe, sel)
            assert_topk_equal(D[i:i + 1], I[i:i + 1], Di, Ii, f"row {i} nprobe={nprobe}")
        Du, Iu = ref.search(x, k, nprobe)     # -1 rows are the unfiltered search
        assert_topk_equal(D[assign < 0], I[assign < 0], Du[assign < 0], Iu[assign < 0], "unfiltered rows")


@pytest.mark.parametrize("explicit", [True, False])
def test_csr_expands_to_the_row_mask(oracle, explicit):
    ref = ragged_ref(oracle, explicit=explicit)
    for name, sel in selectors(ref).items():
        selected = FR.selected_rows(ref, sel)
        for lo, hi in ((0, ref.nlist), (0, 5), (5, ref.nlist), (3, 4)):
            off, blk, word = np_csr(ref.list_len, selected, lo, hi)
            assert len(off) == hi - lo + 1 and (word != 0).all(), name
            for j in range(hi - lo):          # ascending blocks inside each list
                assert (np.diff(blk[off[j]:off[j + 1]].astype(np.int64)) > 0).all(), name
            assert np.array_equal(csr_mask(ref.list_len, off, blk, word, lo, hi), np_mask(ref.list_len, selected, lo, hi)), (name, lo, hi)


def test_doc_label_runs_equal_the_isin_rule():
    from densephrases_b200.mips import MIPS
    rng = np.random.default_rng(8)
    idx_f = synthetic_idx2id([50, 9, 0, 31], rng, ndocs=7)            # random documents: many runs per document
    runs = {}
    for g, n in ((0, 40), (1, 25)):                                    # one run per document, documents out of numeric order
        docs = rng.permutation(12)[:6] + 20
        doc = np.repeat(docs, rng.integers(1, 2 * n // 6, len(docs))).astype(np.int32)
        runs[str(int((g + 7) * 1e9))] = {'doc': doc, 'word': np.zeros(len(doc), np.int32)}
    idx_f.update(runs)
    labels = np.concatenate([int(g) + np.arange(len(t['doc'])) for g, t in idx_f.items()])
    mips = MIPS.from_components(FilterIndexStandIn(labels, 0), idx_f, None, cuda=False, index_path='synthetic_PQ')
    for docs in ([3], [0, 4, 4, 8], [], [100], [25, 21, 3], list(range(40))):
        d = np.unique(np.asarray(docs, dtype=np.int64))
        old = np.concatenate([int(g) + np.flatnonzero(np.isin(t['doc'], d)) for g, t in idx_f.items()] + [np.zeros(0, np.int64)])
        got = mips.doc_labels(docs)
        assert got.dtype == np.int64 and np.array_equal(got, np.sort(old).astype(np.int64)), docs


class QueryFilterStandIn(FilterIndexStandIn):
    """FilterIndexStandIn with per-query filters: a list of selections and the row assignment."""

    def make_query_filters(self, sels, assign=None):
        assign = np.arange(len(sels)) if assign is None else np.asarray(assign)
        return [self.make_filter(s) for s in sels], assign

    def search(self, x, k, filter=None):
        if not isinstance(filter, tuple):
            return super().search(x, k, filter)
        masks, assign = filter
        D = np.empty((len(x), k), np.float32)
        I = np.empty((len(x), k), np.int64)
        for i in range(len(x)):
            D[i:i + 1], I[i:i + 1] = super().search(x[i:i + 1], k, None if assign[i] < 0 else masks[assign[i]])
        return D, I


def test_mips_doc_filters_keep_each_question_in_its_documents():
    from densephrases_b200.mips import MIPS
    rng = np.random.default_rng(9)
    idx_f = synthetic_idx2id([60, 30], rng, ndocs=6)
    labels = np.concatenate([int(g) + np.arange(len(t['doc'])) for g, t in idx_f.items()])
    stand_in = QueryFilterStandIn(labels, 1)
    mips = MIPS.from_components(stand_in, idx_f, None, cuda=False, index_path='synthetic_PQ')
    doc_of = {int(g) + r: int(t['doc'][r]) for g, t in idx_f.items() for r in range(len(t['doc']))}
    per_q = [[1], None, [2, 4], [5]]
    masks, assign = mips.doc_filters(per_q)
    assert list(assign) == [0, -1, 1, 2, 0, -1, 1, 2]             # rows i and B + i share question i's selector
    query = rng.standard_normal((4, 2 * stand_in.d)).astype(np.float32)
    s_doc, _, s_lab, e_doc, _, e_lab, _, _ = mips.search_dense(query, ['q'] * 4, top_k=40, doc_filter=(masks, assign))
    for i, docs in enumerate(per_q):
        for doc, lab in ((s_doc[i], s_lab[i]), (e_doc[i], e_lab[i])):
            assert (doc[lab < 0] == -1).all()
            if docs is not None:
                assert all(doc_of[int(l)] in docs for l in lab[lab >= 0]), i
                assert set(doc[lab >= 0]) <= set(docs)


# ---- both sharded protocols over gloo, local work by the oracle with per-query selections ------------------------------------------
def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from densephrases_b200.sharded import shard_ranges, sharded_search, sharded_search_qsplit
    from oracle import ivfpq_ref as R
    from tests.test_sharded_cpu import _fkey, _fkey_inv
    seed, nlist, nprobe, k = 13, 40, 10, 10
    lens = np.random.default_rng(seed).integers(0, 300, nlist).astype(np.int64)
    ix = R.RefIndex(opq_matrix(seed), R.gen_pq(seed), lens, centroids=R.gen_centroids(seed, 0, nlist), seed=seed)
    x = near_queries(ix, 7, 3)
    rng = np.random.default_rng(seed)
    selected = [(rng.random(ix.ntotal) < p).astype(np.uint8) for p in (0.05, 0.3)]
    assign = np.array([0, -1, 1, 0, 1, -1, 0])
    lo, hi = shard_ranges(lens, world)[rank]
    xr = ix.rotate(x)
    off = np.concatenate([[0], np.cumsum(lens)])
    shard_rows = np.zeros(ix.ntotal, bool)
    shard_rows[off[lo]:off[hi]] = True

    def local(key, xq, kk):
        """This shard's filtered partial top-k of every query (rows of the other shards are never selected), with scan positions."""
        D = np.empty((len(xq), kk), np.float32)
        I = np.empty((len(xq), kk), np.int64)
        G = np.zeros((len(xq), kk), np.int64)
        Cm = ix.centroids()
        for q in range(len(xq)):
            sel = (np.ones(ix.ntotal, np.uint8) if assign[q] < 0 else selected[assign[q]]) & shard_rows
            scores, rows, pos = [], [], []
            start = 0
            lut = R.np_lut(xq[q], ix.pq)
            for l in key[q]:
                l = int(l)
                if l < 0:
                    continue
                if lo <= l < hi and lens[l] > 0:
                    dis0 = R.np_matmul_nt_seq(xq[q:q + 1], Cm[l:l + 1])[0, 0]
                    codes = ix.list_codes(l)
                    dis = np.full(len(codes), dis0, np.float32)
                    for m in range(ix.M):
                        dis = (dis + lut[m, codes[:, m]]).astype(np.float32)
                    scores.append(dis); rows.append(off[l] + np.arange(len(codes))); pos.append(start + np.arange(len(codes)))
                start += lens[l]
            D[q], I[q], G[q] = np.float32(-3.4028234663852886e38), -1, 0
            if scores:
                s, r, p = np.concatenate(scores), np.concatenate(rows), np.concatenate(pos)
                order = np.argsort(-s.astype(np.float64), kind="stable")
                order = order[sel[r[order]].astype(bool)][:kk]
                D[q, :len(order)], I[q, :len(order)], G[q, :len(order)] = s[order], r[order], p[order]
        return torch.from_numpy(D), torch.from_numpy(I), torch.from_numpy(G.astype(np.int32))

    def coarse_local(xt):
        S = R.np_matmul_nt_seq(xr, ix.centroids()[lo:hi])
        keys = np.zeros((len(x), nprobe), dtype=np.uint64)
        for q in range(len(x)):
            order = sorted(range(hi - lo), key=lambda j: (-float(S[q, j]), j))[:nprobe]
            for r, j in enumerate(order):
                keys[q, r] = (_fkey(S[q, j]) << np.uint64(32)) | np.uint64(0xFFFFFFFF - (j + lo))
        return torch.from_numpy(keys.view(np.int64))

    def search_preassigned(keys_g, kk):
        kg = keys_g.numpy().view(np.uint64)
        key = np.full((len(x), nprobe), -1, dtype=np.int64)
        for q in range(len(x)):
            allk = sorted((int(v) for v in kg[:, q, :].ravel() if v != 0), reverse=True)[:nprobe]
            key[q, :len(allk)] = [0xFFFFFFFF - (v & 0xFFFFFFFF) for v in allk]
        return local(key, xr, kk)

    def pack(D, I, G):
        ck = (_fkey(D.numpy()) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - (G.numpy().astype(np.int64) & 0xFFFFFFFF).astype(np.uint64))
        return torch.from_numpy(np.ascontiguousarray(np.stack([np.where(I.numpy() >= 0, ck, 0).view(np.int64), I.numpy()], axis=-1)))

    def merge_packed(Pg, kk):
        Pn = Pg.numpy()
        D = np.full((len(x), kk), np.float32(-3.4028234663852886e38), dtype=np.float32)
        I = np.full((len(x), kk), -1, dtype=np.int64)
        for q in range(len(x)):
            ent = sorted(((int(np.uint64(Pn[s, q, r, 0])), int(Pn[s, q, r, 1])) for s in range(Pn.shape[0]) for r in range(kk)
                          if Pn[s, q, r, 0] != 0), reverse=True)[:kk]
            for i, (ckey, lab) in enumerate(ent):
                D[q, i], I[q, i] = _fkey_inv(ckey >> 32), lab
        return torch.from_numpy(D), torch.from_numpy(I)

    Dm, Im = sharded_search(torch.from_numpy(x), k, world, None, coarse_local, search_preassigned, pack, merge_packed)
    R_ = 768 + 2 * nprobe

    def coarse_split(xl):
        xrl = ix.rotate(xl.numpy())
        S = R.np_matmul_nt_seq(xrl, ix.centroids())
        rec = np.zeros((len(xrl), R_), dtype=np.float32)
        for q in range(len(xrl)):
            order = sorted(range(nlist), key=lambda j: (-float(S[q, j]), j))[:nprobe]
            rec[q, :768] = xrl[q]
            rec[q, 768:768 + nprobe] = np.array(order, dtype=np.int32).view(np.float32)
            rec[q, 768 + nprobe:] = S[q, order]
        return torch.from_numpy(rec)

    def search_assigned(rec_g, kk):
        rec = rec_g.numpy()
        key = np.ascontiguousarray(rec[:, 768:768 + nprobe]).view(np.int32).astype(np.int64)
        return local(key, np.ascontiguousarray(rec[:, :768]), kk)

    Dq, Iq = sharded_search_qsplit(torch.from_numpy(x), k, world, rank, None, coarse_split, search_assigned, pack, merge_packed)
    if rank == 0:
        Dw, Iw = query_filtered_search(ix, x, k, nprobe, selected, assign)
        np.savez(out, D=Dm.numpy(), I=Im.numpy(), Dq=Dq.numpy(), Iq=Iq.numpy(), Dw=Dw, Iw=Iw)
    dist.destroy_process_group()


def test_gloo_world2_both_protocols_with_per_query_selections(tmp_path, oracle):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "qf2.npz")
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    g = np.load(out)
    assert_topk_equal(g["D"], g["I"], g["Dw"], g["Iw"], "two-exchange protocol vs the per-query definition")
    assert_topk_equal(g["Dq"], g["Iq"], g["Dw"], g["Iw"], "query-split protocol vs the per-query definition")
