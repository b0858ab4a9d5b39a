"""Index builder: train and fill an OPQ96 / IVF{nlist} / PQ96 inner-product phrase index without FAISS.

Restates what reference build_phrase_index.py asks faiss to do (SURVEY.md 8f #4; offline, not on the serving hot path):
  train_index  (:96-142)   IndexPreTransform(OPQMatrix(768, 96; niter=10), IndexIVFPQ(IndexFlatIP(768), 768, nlist, 96, 8, IP))
  add_to_index (:145-150)  add_with_ids(vectors, ids = arange + offset + running_total)
following the published faiss algorithms: OPQ (Ge et al., non-parametric variant: alternate PQ training with an orthogonal
Procrustes update of the rotation), k-means coarse quantizer with inner-product assignment (an IVF index over IndexFlatIP assigns
each vector to the centroid of MAXIMUM inner product), PQ trained on RESIDUALS (by_residual=True) and encoded by nearest codeword
in L2 per 8-dim sub-vector.  Plain PyTorch (CPU or CUDA) -- this is an offline tool; its outputs are exactly the arrays
IvfPqIndex.from_arrays consumes.  Randomness is seeded; faiss' own random initialisations are not reproduced (trained indexes are
equivalent in kind, not bit-identical to a faiss-trained one).

Training on the GPU (index.train of build_phrase_index.py:96-142, with the fixed fp32 order of DESIGN.md 3.3; train_index_gpu below):
    ix = IvfPqIndex(nlist)
    ix.train(x_train)                            # OPQ, spherical k-means coarse quantizer, PQ on residuals -> trained, empty
    ix.add_with_ids(x, ids)                      # as below
    list_len, codes, ids = ix.lists()
    artifacts.write_faiss_index(path, ix.opq_matrix(), ix.centroids(), ix.pq_codebooks(), list_len, codes, ids)
Filling an index on the GPU (the add_with_ids of build_phrase_index.py:145-150,156-279, with the exact fp32 encoding of DESIGN.md 3.1):
    A, centroids, pq = train_index(x_train, nlist)
    ix = IvfPqIndex.from_arrays(A, centroids, pq, np.zeros(nlist, np.int64), np.zeros((0, 96), np.uint8))   # trained, empty
    for x, ids in chunks:                        # numpy or CUDA tensors; ids None -> ntotal + arange(n)
        ix.add_with_ids(x, ids)
    list_len, codes, ids = ix.lists()            # list-major, what set_lists takes
    artifacts.write_faiss_index(path, A, centroids, pq, list_len, codes, ids)
Updating a document (DESIGN.md 3.2): its phrases carry consecutive labels [first, first + n) (build_phrase_index.py:149), so
    ix.remove_ids(range(first, first + n))       # faiss remove_ids(IDSelectorRange); a label array drops a set of documents
    ix.add_with_ids(x_new, ids_new)              # the document's new phrase vectors
Keeping idx2id and the phrase metadata in step with re-added documents is the caller's job.
Merging sub-indexes (the merge stage of build_phrase_index.py:282-338, DESIGN.md 3.4), e.g. one read from a %d.faiss file:
    sub = artifacts.read_faiss_index(path)       # same OPQ matrix, centroids and PQ codebooks as ix
    ix.merge_from(IvfPqIndex.from_arrays(sub["A"], sub["centroids"], sub["pq"], sub["list_len"], sub["codes"], sub["ids"]))
    # several at once: ix.merge_from([a, b, c], add_id=offset) appends them in order, labels + offset; the sources stay as they were
add_to_index below is the PyTorch encoder that runs without a GPU; its argmax / argmin have no fixed floating-point order, so on
ties and near-ties it may pick other lists or codewords than IvfPqIndex.encode."""
import logging
import os
import pickle
import random
import time

import numpy as np
import torch

D, M, KSUB, DSUB = 768, 96, 256, 8
logger = logging.getLogger(__name__)


def _kmeans(x, k, niter, seed, assign_ip=False):
    """Lloyd's k-means; assignment by max inner product (coarse quantizer over IndexFlatIP) or min L2 (PQ codebooks)."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    n = x.shape[0]
    cent = x[torch.randperm(n, generator=g)[:k].to(x.device)].clone()
    if cent.shape[0] < k:                                   # fewer points than centroids: pad with jittered copies
        extra = cent[torch.randint(0, cent.shape[0], (k - cent.shape[0],), generator=g).to(x.device)]
        cent = torch.cat([cent, extra + 1e-4 * torch.randn(extra.shape, generator=g).to(x.device)])
    for _ in range(niter):
        if assign_ip:
            a = (x @ cent.T).argmax(1)
        else:
            a = (cent.pow(2).sum(1)[None, :] - 2.0 * (x @ cent.T)).argmin(1)
        sums = torch.zeros_like(cent).index_add_(0, a, x)
        cnt = torch.zeros(k, device=x.device).index_add_(0, a, torch.ones(n, device=x.device))
        alive = cnt > 0
        cent[alive] = sums[alive] / cnt[alive, None]
        if (~alive).any():                                  # faiss splits big clusters to re-seed empty ones; re-seed from data here
            idx = torch.randint(0, n, (int((~alive).sum()),), generator=g).to(x.device)
            cent[~alive] = x[idx]
    return cent


def _train_pq(res, niter, seed):
    """-> codebooks [M, 256, 8] trained independently per sub-space on residual vectors [n, 768]."""
    books = []
    for m in range(M):
        books.append(_kmeans(res[:, m * DSUB:(m + 1) * DSUB].contiguous(), KSUB, niter, seed + 101 * m))
    return torch.stack(books)


def _pq_encode(res, pq):
    codes = torch.empty((res.shape[0], M), dtype=torch.uint8, device=res.device)
    for m in range(M):
        sub = res[:, m * DSUB:(m + 1) * DSUB]
        cb = pq[m]
        codes[:, m] = (cb.pow(2).sum(1)[None, :] - 2.0 * (sub @ cb.T)).argmin(1).to(torch.uint8)
    return codes


def _pq_decode(codes, pq):
    return torch.cat([pq[m][codes[:, m].long()] for m in range(M)], dim=1)


def train_index(x, nlist, niter_opq=10, niter_km=10, niter_pq=8, seed=123, device=None):
    """x [ns, 768] float32 training sample -> (A [768,768] OPQ rotation (xr = x A^T), centroids [nlist,768], pq [96,256,8])."""
    dev = torch.device(device) if device else torch.device('cpu')
    x = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).to(dev)
    g = torch.Generator().manual_seed(seed)
    A = torch.linalg.qr(torch.randn((D, D), generator=g))[0].to(dev)              # random orthonormal start (faiss OPQMatrix::train)
    for it in range(niter_opq):
        xr = x @ A.T
        pq0 = _train_pq(xr, max(niter_pq // 2, 2), seed + it)
        y = _pq_decode(_pq_encode(xr, pq0), pq0)                                   # best PQ approximation in the rotated space
        u, _, vt = torch.linalg.svd(x.T @ y, full_matrices=False)                   # Procrustes: R = U V^T maximises tr(R^T X^T Y)
        A = (u @ vt).T.contiguous()
    xr = x @ A.T
    centroids = _kmeans(xr, nlist, niter_km, seed + 7, assign_ip=True)
    assign = (xr @ centroids.T).argmax(1)
    pq = _train_pq(xr - centroids[assign], niter_pq, seed + 13)
    return A.cpu().numpy(), centroids.cpu().numpy(), pq.cpu().numpy()


def train_index_gpu(x, nlist, niter_opq=10, niter_km=10, niter_pq=25, seed=123, max_points_per_centroid=256, device=0):
    """train_index on the GPU (IvfPqIndex.train): x [ns, 768] numpy or CUDA float32 -> (A, centroids, pq) like train_index.  Unlike
    train_index it subsamples to max_points_per_centroid per centroid, so it trains the IVF65536 and larger shapes, and its coarse
    k-means is spherical, as faiss' is for an inner-product IVF index."""
    from .ivfpq import IvfPqIndex
    ix = IvfPqIndex(nlist, device=device)
    ix.train(x, niter=niter_km, niter_pq=niter_pq, opq_niter=niter_opq, seed=seed, max_points_per_centroid=max_points_per_centroid)
    return ix.opq_matrix(), ix.centroids(), ix.pq_codebooks()


def add_to_index(A, centroids, pq, x, ids=None, offset=0, running_total=0, device=None, chunk=65536):
    """Assign + encode vectors x [n,768].  -> (list_no [n] int64, codes [n,96] uint8, ids [n] int64) in input order.
    ids default to arange + offset + running_total (build_phrase_index.py:149-150)."""
    dev = torch.device(device) if device else torch.device('cpu')
    At, Ct, Pt = (torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dev) for a in (A, centroids, pq))
    x = np.ascontiguousarray(x, dtype=np.float32)
    list_no = np.empty(len(x), dtype=np.int64)
    codes = np.empty((len(x), M), dtype=np.uint8)
    for s in range(0, len(x), chunk):
        xr = torch.from_numpy(x[s:s + chunk]).to(dev) @ At.T
        a = (xr @ Ct.T).argmax(1)
        list_no[s:s + chunk] = a.cpu().numpy()
        codes[s:s + chunk] = _pq_encode(xr - Ct[a], Pt).cpu().numpy()
    if ids is None:
        ids = np.arange(len(x), dtype=np.int64) + offset + running_total
    return list_no, codes, np.asarray(ids, dtype=np.int64)


def to_list_major(list_no, codes, ids, nlist):
    """Group (list_no, codes, ids) by inverted list, keeping insertion order inside a list (what faiss' ArrayInvertedLists holds).
    -> (list_len [nlist], codes, ids) ready for IvfPqIndex.from_arrays / set_lists."""
    order = np.argsort(list_no, kind='stable')
    return np.bincount(list_no, minlength=nlist).astype(np.int64), codes[order], ids[order]


def build_index(x_train, x_add, nlist, ids=None, seed=123, device=None, **train_kw):
    """Convenience: train on x_train, add x_add -> dict(A, centroids, pq, list_len, codes, ids)."""
    A, centroids, pq = train_index(x_train, nlist, seed=seed, device=device, **train_kw)
    list_no, codes, ids = add_to_index(A, centroids, pq, x_add, ids=ids, device=device)
    list_len, codes, ids = to_list_major(list_no, codes, ids, nlist)
    return dict(A=A, centroids=centroids, pq=pq, list_len=list_len, codes=codes, ids=ids)


def save_container(path, index_arrays):
    """Write the `index.dph.npz` container MIPS.__init__ reads (next to where the reference expects index.faiss)."""
    np.savez(path, **index_arrays)


# ---------------------------------------------------------------------------------------------------------------------------------
# build_phrase_index.py over a phrase dump (DESIGN.md 3.8): the stages coarse / fine / all / add / merge of run_index (:341-405)
# ---------------------------------------------------------------------------------------------------------------------------------
NO_FILTER = -1e8


def int8_to_float(q, offset, scale):
    """The reference's int8_to_float (embed_utils.py:148-149) as numpy 1.x computed it: the group's float64 offset and scale attributes
    become fp32 under value-based casting, and the arithmetic is fp32, fl32(fl32(float(q) / scale) + offset).  Numpy 2 would compute
    in float64; this keeps the fp32 chain.  IvfPqIndex.add_int8 computes the same values on the device."""
    return np.asarray(q).astype(np.float32) / np.float32(scale) + np.float32(offset)


def get_args(argv=None):
    """build_phrase_index.py:get_args (:19-44): the reference's flags (Options.add_index_options) and the paths derived from them."""
    from .options import Options
    options = Options()
    options.add_index_options()
    return derive_paths(options.parse(argv))


def derive_paths(args):
    """index_name = <num_clusters>_flat_<fine_quant>[_first][_ft<int>], index_dir = dump_dir/start/<index_name>, and the file paths in
    it; with --dump_paths the sub-index paths index/<offset>.faiss and index/<offset>.hdf5 and the dump paths under phrase_dir."""
    coarse = 'hnsw' if args.hnsw else 'flat'
    args.index_name = f'{args.num_clusters}_{coarse}_{args.fine_quant}{"_first" if args.first_passage else ""}'
    if args.index_filter != NO_FILTER:
        args.index_name = args.index_name + f'_ft{int(args.index_filter)}'
    args.index_dir = os.path.join(args.dump_dir, 'start', args.index_name)
    args.quantizer_path = os.path.join(args.index_dir, args.quantizer_path)
    args.trained_index_path = os.path.join(args.index_dir, args.trained_index_path)
    args.inv_path = os.path.join(args.index_dir, args.inv_path)
    args.subindex_dir = os.path.join(args.index_dir, args.subindex_name)
    if args.dump_paths is None:
        args.index_path = os.path.join(args.index_dir, args.index_path)
        args.idx2id_path = os.path.join(args.index_dir, args.idx2id_path)
    else:
        args.dump_paths = [os.path.join(args.dump_dir, args.phrase_dir, path) for path in args.dump_paths.split(',')]
        args.index_path = os.path.join(args.subindex_dir, '%d.faiss' % args.offset)
        args.idx2id_path = os.path.join(args.subindex_dir, '%d.hdf5' % args.offset)
    return args


class _Dump(object):
    """One dump file through artifacts' HDF5 reader: its documents in the group B-tree's byte-wise name order, which is the order
    h5py yields them in ("10" before "2")."""

    def __init__(self, path):
        from . import artifacts
        self.h = artifacts.open_hdf5(path)
        self.docs = list(self.h.children(self.h.root_addr).items())

    def members(self, addr):
        return self.h.children(addr)

    def dataset(self, members, name):
        return self.h.dataset(members[name])


def sample_data(dump_paths, doc_sample_ratio=0.2, vec_sample_ratio=0.2, seed=29, norm_th=999):
    """build_phrase_index.py:sample_data (:60-93): random.sample of the documents of each file and np.random.choice (with replacement)
    of the rows of each sampled document, both seeded once with 29, dequantised in fp32 and cut at fp32 norm <= norm_th.
    -> (sample [n, 768] f32, avg_vec [1, 768], std_vec [1, 768])."""
    random.seed(seed)
    np.random.seed(seed)
    out = []
    for path in dump_paths:
        f = _Dump(path)
        doc_ids = [name for name, _ in f.docs]
        addr = dict(f.docs)
        for doc_id in random.sample(doc_ids, int(doc_sample_ratio * len(doc_ids))):
            members = f.members(addr[doc_id])
            start = f.dataset(members, 'start')
            if len(start.shape) < 2 or start.shape[0] == 0:
                continue
            idx = np.random.choice(start.shape[0], int(vec_sample_ratio * start.shape[0]))
            attrs = f.h.attributes(addr[doc_id])
            vec = int8_to_float(start, attrs['offset'], attrs['scale'])[idx]
            out.append(vec[np.linalg.norm(vec, axis=1) <= norm_th])
    x = np.concatenate(out) if out else np.zeros((0, D), np.float32)
    return x, np.mean(x, axis=0, keepdims=True), np.std(x, axis=0, keepdims=True)


def train_phrase_index(x, num_clusters, trained_index_path, device=0):
    """train_index (:96-142) for OPQ96: IvfPqIndex.train (faiss' recipe, DESIGN.md 3.3), written as trained.faiss with empty lists."""
    from . import artifacts
    from .ivfpq import IvfPqIndex
    if len(x) < max(num_clusters, KSUB):
        raise ValueError(f'the training sample holds {len(x)} vectors; training IVF{num_clusters} with PQ96 needs at least '
                         f'max(num_clusters, 256) = {max(num_clusters, KSUB)} (raise doc_sample_ratio / vec_sample_ratio)')
    ix = IvfPqIndex(num_clusters, device=device)
    ix.train(np.ascontiguousarray(x, dtype=np.float32))
    artifacts.write_faiss_index(trained_index_path, ix.opq_matrix(), ix.centroids(), ix.pq_codebooks(), np.zeros(num_clusters, np.int64),
                                np.zeros((0, M), np.uint8), np.zeros(0, np.int64))


def _trained_index(trained_index_path, device=0):
    from . import artifacts
    from .ivfpq import IvfPqIndex
    t = artifacts.read_faiss_index(trained_index_path)
    return t, IvfPqIndex.from_arrays(t['A'], t['centroids'], t['pq'], np.zeros(len(t['list_len']), np.int64), np.zeros((0, M), np.uint8),
                                     device=device)


def pinned_rows(n):
    """A page-locked int8 [n, 768] numpy array (add_int8 reads it in place through its device mapping)."""
    return torch.empty((n, D), dtype=torch.int8).pin_memory().numpy()


class _Adder(object):
    """Gathers the int8 rows of about num_docs_per_add documents into one reused page-locked buffer and hands each run of documents
    with the same (offset, scale) to add_int8, labels offset + running total.  Host memory stays one batch."""

    def __init__(self, ix, label0, timings):
        self.ix, self.next_label, self.t = ix, label0, timings
        self.pending, self.buf = [], None

    def push(self, rows, offset, scale):
        self.pending.append((rows, float(offset), float(scale)))

    def flush(self):
        runs, i = [], 0
        while i < len(self.pending):
            j = i
            while j < len(self.pending) and self.pending[j][1:] == self.pending[i][1:]:
                j += 1
            runs.append((self.pending[i:j], self.pending[i][1], self.pending[i][2]))
            i = j
        self.pending = []
        for docs, offset, scale in runs:
            n = sum(len(r) for r, _, _ in docs)
            if n == 0:
                continue
            t0 = time.perf_counter()
            if self.buf is None or len(self.buf) < n:
                self.buf = pinned_rows(max(n, 2 * len(self.buf) if self.buf is not None else n))
            at = 0
            for r, _, _ in docs:
                self.buf[at:at + len(r)] = r
                at += len(r)
            t1 = time.perf_counter()
            self.ix.add_int8(self.buf[:n], np.arange(self.next_label, self.next_label + n, dtype=np.int64), offset, scale)
            t2 = time.perf_counter()
            self.next_label += n
            self.t['gather'] = self.t.get('gather', 0.0) + t1 - t0
            self.t['add'] = self.t.get('add', 0.0) + t2 - t1
            self.t['rows'] = self.t.get('rows', 0) + n
            self.t['h2d_bytes'] = self.t.get('h2d_bytes', 0) + n * D


def add_dump_to_index(dump_paths, trained_index_path, target_index_path, idx2id_path, num_docs_per_add=1000, offset=0,
                 first_passage=False, index_filter=NO_FILTER, device=0, timings=None):
    """build_phrase_index.py:add_to_index (:156-279) for OPQ96 on the GPU: every document with rows, in the dumps' order and each file's
    h5py order, its rows cut to the first passage (f2o_start < len_per_para[0]) or to the rows the filter dump keeps (index_filter),
    added through add_int8 with labels offset + running total.  Writes target_index_path (the trained tables and the lists) and
    idx2id_path ({str(offset): doc, word int32, attrs offset}).  -> the IvfPqIndex.  The reference computes norms against norm_th
    here but adds every row, and so does this."""
    from . import artifacts
    timings = {} if timings is None else timings
    t, ix = _trained_index(trained_index_path, device)
    adder = _Adder(ix, offset, timings)
    doc_out, word_out = [], []
    for path in dump_paths:
        t0 = time.perf_counter()
        f = _Dump(path)
        ff = _Dump(path.replace('/phrase/', '/filter/')) if index_filter != NO_FILTER else None
        faddr = dict(ff.docs) if ff is not None else None
        last = len(f.docs) - 1
        for i, (doc_idx, addr) in enumerate(f.docs):
            members = f.members(addr)
            start = f.dataset(members, 'start')
            if start.shape[0] == 0:
                continue
            attrs = f.h.attributes(addr)
            if first_passage:
                f2o = f.dataset(members, 'f2o_start')
                cut = int((f2o < f.dataset(members, 'len_per_para')[0]).sum())
                start, words = start[:cut], np.arange(cut)
            elif index_filter != NO_FILTER:
                fm = ff.members(faddr[doc_idx])
                fs, fe = ff.dataset(fm, 'filter_start'), ff.dataset(fm, 'filter_end')
                o2f = {orig: ft for ft, orig in enumerate(f.dataset(members, 'f2o_start').tolist())}
                keep = set(np.concatenate([np.where(fs > index_filter)[0], np.where(fe > index_filter)[0]]).tolist())
                words = np.asarray(sorted(o2f[si] for si in keep if si in o2f), dtype=np.int64)
                start = start[words]
            else:
                words = np.arange(len(start))
            adder.push(start, attrs['offset'], attrs['scale'])
            doc_out.append(np.full(len(start), int(doc_idx), dtype=np.int32))
            word_out.append(words.astype(np.int32))
            if i % num_docs_per_add == 0 or i == last:
                timings['read'] = timings.get('read', 0.0) + time.perf_counter() - t0
                adder.flush()
                t0 = time.perf_counter()
        timings['read'] = timings.get('read', 0.0) + time.perf_counter() - t0
        adder.flush()
    t0 = time.perf_counter()
    list_len, codes, ids = ix.lists()
    artifacts.write_faiss_index(target_index_path, t['A'], t['centroids'], t['pq'], list_len, codes, ids)
    doc = np.concatenate(doc_out) if doc_out else np.zeros(0, np.int32)
    word = np.concatenate(word_out) if word_out else np.zeros(0, np.int32)
    artifacts.write_hdf5(idx2id_path, {str(offset): {'doc': doc, 'word': word}}, attrs={str(offset): {'offset': int(offset)}})
    timings['write'] = timings.get('write', 0.0) + time.perf_counter() - t0
    return ix


def merge_indexes(subindex_dir, trained_index_path, target_index_path, target_idx2id_path, target_inv_path):
    """build_phrase_index.py:merge_indexes (:282-338) without a GPU: each list holds the sub-indexes' entries of that list in source
    order (faiss OnDiskInvertedLists.merge_from), written as index.faiss with its lists in the side file target_inv_path, and the
    idx2id groups of every sub-index in one idx2id.hdf5.  The sub-indexes are taken in ascending offset order; the reference takes
    os.listdir's order, which depends on the file system.  A sub-index whose OPQ matrix, centroids or PQ codebooks differ in any bit
    from trained.faiss is rejected."""
    from . import artifacts
    names = os.listdir(subindex_dir)
    offsets = sorted(int(n[:-len('.faiss')]) for n in names if n.endswith('.faiss'))
    if sorted(int(n[:-len('.hdf5')]) for n in names if n.endswith('.hdf5')) != offsets:
        raise ValueError(f'{subindex_dir}: the .faiss and .hdf5 sub-index files do not pair up')
    t = artifacts.read_faiss_index(trained_index_path)
    nlist = len(t['list_len'])
    list_no, codes, ids, idx2id = [], [], [], {}
    for off in offsets:
        sub = artifacts.read_faiss_index(os.path.join(subindex_dir, '%d.faiss' % off))
        for key in ('A', 'centroids', 'pq'):
            if sub[key].shape != t[key].shape or not np.array_equal(sub[key].view(np.uint32), t[key].view(np.uint32)):
                raise ValueError(f'{off}.faiss: its {key} is not bit-identical to {trained_index_path}')
        list_no.append(np.repeat(np.arange(nlist, dtype=np.int64), sub['list_len']))
        codes.append(sub['codes']); ids.append(sub['ids'])
        for key, g in artifacts.read_idx2id(os.path.join(subindex_dir, '%d.hdf5' % off)).items():
            if key in idx2id:
                raise ValueError(f'idx2id group {key} appears in two sub-indexes')
            idx2id[key] = g
    list_len, codes, ids = to_list_major(np.concatenate(list_no + [np.zeros(0, np.int64)]),
                                         np.concatenate(codes + [np.zeros((0, M), np.uint8)]),
                                         np.concatenate(ids + [np.zeros(0, np.int64)]), nlist)
    artifacts.write_faiss_index(target_index_path, t['A'], t['centroids'], t['pq'], list_len, codes, ids,
                                ondisk_payload=os.path.basename(target_inv_path))
    artifacts.write_hdf5(target_idx2id_path, {k: {'doc': g['doc'], 'word': g['word']} for k, g in idx2id.items()},
                         attrs={k: {'offset': int(k)} for k in idx2id})
    return list_len, codes, ids


def check_args(args):
    """The refusals of this builder: it builds the OPQ96 / IVF-flat index only (DESIGN.md 0) and has no `move` stage."""
    if args.stage not in ('all', 'coarse', 'fine', 'add', 'merge'):
        raise ValueError(f'--stage {args.stage!r}: this builder runs all, coarse, fine, add and merge (move is not supported)')
    if args.fine_quant != 'OPQ96' or args.hnsw:
        raise ValueError(f'--fine_quant {args.fine_quant}{" --hnsw" if args.hnsw else ""}: only the OPQ96 IVF-flat index '
                         '(--fine_quant OPQ96, no --hnsw) is supported; SQ4, flat ("none") and HNSW indexes are not')
    if args.first_passage and args.index_filter != NO_FILTER:
        raise ValueError('--first_passage and --index_filter together: the reference fails on this combination; pass one of them')


def run_index(args, device=0, timings=None):
    """build_phrase_index.py:run_index (:341-405) on the GPU (with or without --cuda; there is no CPU path) for args from get_args.
    Stage `fine` on its own draws the sample again (the reference fails there with UnboundLocalError and an unexpected hnsw= keyword
    of sample_data).  Files that exist are kept unless --replace, as in the reference.  timings (dict): seconds of each stage."""
    check_args(args)
    timings = {} if timings is None else timings
    phrase_dir = os.path.join(args.dump_dir, args.phrase_dir)
    names = os.listdir(phrase_dir) if os.path.isdir(phrase_dir) else []
    dump_paths = sorted(os.path.join(phrase_dir, n) for n in names if n.endswith('.hdf5'))
    sample = None

    def draw():
        t0 = time.perf_counter()
        out = sample_data(dump_paths, args.doc_sample_ratio, args.vec_sample_ratio, norm_th=args.norm_th)
        timings['sample'] = timings.get('sample', 0.0) + time.perf_counter() - t0
        return out

    # The reference never writes quantizer_path for OPQ indexes, so `all` and `coarse` always draw the sample.
    if args.stage in ('all', 'coarse') and (args.replace or not os.path.exists(args.quantizer_path)):
        os.makedirs(args.index_dir, exist_ok=True)
        sample, avg_vec, std_vec = draw()
        with open(os.path.join(args.index_dir, 'avg_vec.pkl'), 'wb') as fp:
            pickle.dump(avg_vec, fp)
        with open(os.path.join(args.index_dir, 'std_vec.pkl'), 'wb') as fp:
            pickle.dump(std_vec, fp)
    if args.stage in ('all', 'fine') and (args.replace or not os.path.exists(args.trained_index_path)):
        os.makedirs(args.index_dir, exist_ok=True)
        if sample is None:
            sample = draw()[0]
        t0 = time.perf_counter()
        train_phrase_index(sample, args.num_clusters, args.trained_index_path, device)
        timings['train'] = time.perf_counter() - t0
    if args.stage in ('all', 'add') and (args.replace or not os.path.exists(args.index_path)):
        if args.dump_paths is not None:
            dump_paths = args.dump_paths
            os.makedirs(args.subindex_dir, exist_ok=True)
        add_dump_to_index(dump_paths, args.trained_index_path, args.index_path, args.idx2id_path, num_docs_per_add=args.num_docs_per_add,
                     offset=args.offset, first_passage=args.first_passage, index_filter=args.index_filter, device=device, timings=timings)
    if args.stage == 'merge' and (args.replace or not os.path.exists(args.index_path)):
        t0 = time.perf_counter()
        merge_indexes(args.subindex_dir, args.trained_index_path, args.index_path, args.idx2id_path, args.inv_path)
        timings['merge'] = time.perf_counter() - t0
    return timings


def main(argv=None):
    logging.basicConfig(format='%(asctime)s - %(levelname)s - %(name)s -   %(message)s', level=logging.INFO)
    run_index(get_args(argv))


if __name__ == '__main__':
    main()
