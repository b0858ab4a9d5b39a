#!/usr/bin/env python
"""Convert a DensePhrases release (index.faiss + idx2id.hdf5 + meta_compressed.pkl) into the containers densephrases_b200.MIPS reads
(index.dph.npz + idx2id.npz + meta_dph.pkl).  Run this ONCE on a machine that still has the reference's dependencies
(faiss, h5py, blosc -- requirements.txt of princeton-nlp/DensePhrases); the GPU serving path itself needs none of them.

    python tools/convert_reference_artifacts.py $SAVE_DIR/densephrases-multi_wiki-20181220/dump start/1048576_flat_OPQ96 [--verify]

--verify additionally parses the same three files with the library-free readers of densephrases_b200/artifacts.py and checks that
they return exactly what faiss / h5py / blosc returned: that is the cross-check those readers still need (they were written without
access to the libraries or to any file produced by them).

It only uses public faiss Python API calls (the same ones densephrases/index.py:30-32,52 and build_phrase_index.py use);
it cannot be exercised in the offline build image (no faiss there), so treat it as a recipe: untested against a real release."""
import os
import pickle
import sys
import zlib

import numpy as np


def convert_index(index_path, out_path):
    import faiss
    index = faiss.read_index(index_path)                                               # IndexPreTransform(OPQMatrix, IndexIVFPQ)
    d = index.d
    A = faiss.vector_to_array(faiss.downcast_VectorTransform(index.chain.at(0)).A).reshape(d, d).astype(np.float32)   # index.py:32
    ivf = faiss.downcast_index(faiss.extract_index_ivf(index))                           # IndexIVFPQ
    assert ivf.pq.M == 96 and ivf.pq.nbits == 8 and ivf.by_residual, "only OPQ96 / PQ96 x 8 bit, by_residual (build_phrase_index.py:113-116)"
    nlist = ivf.nlist
    quantizer = faiss.downcast_index(ivf.quantizer)                                      # IndexFlatIP
    centroids = faiss.vector_to_array(quantizer.xb).reshape(nlist, d).astype(np.float32)
    pq = faiss.vector_to_array(ivf.pq.centroids).reshape(ivf.pq.M, ivf.pq.ksub, ivf.pq.dsub).astype(np.float32)
    inv = ivf.invlists
    list_len = np.array([inv.list_size(l) for l in range(nlist)], dtype=np.int64)
    codes = np.empty((int(list_len.sum()), inv.code_size), dtype=np.uint8)
    ids = np.empty(int(list_len.sum()), dtype=np.int64)
    o = 0
    for l in range(nlist):
        n = int(list_len[l])
        if n:
            codes[o:o + n] = faiss.rev_swig_ptr(inv.get_codes(l), n * inv.code_size).reshape(n, inv.code_size)
            ids[o:o + n] = faiss.rev_swig_ptr(inv.get_ids(l), n)
            o += n
    np.savez(out_path, A=A, centroids=centroids, pq=pq, list_len=list_len, codes=codes, ids=ids)
    print(f"{out_path}: ntotal {o}, nlist {nlist}")


def convert_idx2id(h5_path, out_path):
    import h5py
    out = {}
    with h5py.File(h5_path, "r") as f:                                                   # groups str(offset) -> doc, word (build_phrase_index.py:268-276)
        for key in f:
            out[f"{key}/doc"] = f[key]["doc"][:]
            out[f"{key}/word"] = f[key]["word"][:]
    np.savez(out_path, **out)


def convert_meta(pkl_path, out_path):
    import blosc
    src = pickle.load(open(pkl_path, "rb"))                                              # compress_metadata.py:32-53,108-111
    dst = {}
    for doc_id, g in src.items():
        rec = {"title": g["title"], "dtypes": g["dtypes"]}
        for name in ("word2char_start", "word2char_end", "f2o_start"):
            rec[name] = zlib.compress(blosc.decompress(g[name]))
        rec["context"] = zlib.compress(blosc.decompress(g["context"]))
        dst[doc_id] = rec
    pickle.dump(dst, open(out_path, "wb"))


def verify(dump_dir, index_dir):
    """Native readers (densephrases_b200/artifacts.py) against what the libraries produced above."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from densephrases_b200 import artifacts
    want = np.load(os.path.join(index_dir, "index.dph.npz"))
    got = artifacts.read_faiss_index(os.path.join(index_dir, "index.faiss"))
    for k in ("A", "centroids", "pq", "list_len", "codes", "ids"):
        assert np.array_equal(got[k], want[k]), f"index.faiss: {k} differs between faiss and the native reader"
    want = np.load(os.path.join(index_dir, "idx2id.npz"))
    got = artifacts.read_idx2id(os.path.join(index_dir, "idx2id.hdf5"))
    assert sorted(f"{k}/{t}" for k in got for t in got[k]) == sorted(want.files), "idx2id.hdf5: group names differ"
    for member in want.files:
        key, kind = member.split("/")
        assert np.array_equal(got[key][kind], want[member]), f"idx2id.hdf5: {member} differs"
    meta = os.path.join(dump_dir, "meta_compressed.pkl")
    if os.path.exists(meta):
        import blosc
        src = pickle.load(open(meta, "rb"))
        for n, (doc_id, g) in enumerate(src.items()):
            for name in ("word2char_start", "word2char_end", "f2o_start", "context"):
                assert artifacts.blosc_decompress(g[name]) == blosc.decompress(g[name]), f"meta_compressed.pkl: {doc_id}/{name} differs"
            if n >= 2000:
                break
    print("native readers agree with faiss / h5py / blosc")


if __name__ == "__main__":
    do_verify = "--verify" in sys.argv
    args = [a for a in sys.argv[1:] if a != "--verify"]
    dump_dir, index_name = args[0], args[1]
    index_dir = os.path.join(dump_dir, index_name)
    convert_index(os.path.join(index_dir, "index.faiss"), os.path.join(index_dir, "index.dph.npz"))
    convert_idx2id(os.path.join(index_dir, "idx2id.hdf5"), os.path.join(index_dir, "idx2id.npz"))
    meta = os.path.join(dump_dir, "meta_compressed.pkl")
    if os.path.exists(meta):
        convert_meta(meta, os.path.join(dump_dir, "meta_dph.pkl"))
    if do_verify:
        verify(dump_dir, index_dir)
