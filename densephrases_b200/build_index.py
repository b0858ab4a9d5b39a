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
import numpy as np
import torch

D, M, KSUB, DSUB = 768, 96, 256, 8


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
