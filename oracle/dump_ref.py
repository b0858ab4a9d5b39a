"""oracle/dump_ref.py -- TEST INFRASTRUCTURE.  Plain numpy restatement of one document's numeric dump fields as the reference's
get_metadata -> filter_metadata -> compress_metadata compute them (densephrases/utils/embed_utils.py:40-191) from fp32 inputs:
the kept rows (union of filter_start > thr and filter_end > thr), their int8 vectors, f2o_start and start2end re-indexed to the
kept rows.  tests/test_dump_cpu.py pins it against the unmodified reference (tests/golden/dump_reference.json.gz)."""
import numpy as np


def select_document(start, filter_start, filter_end, rows_per_feature, max_answer_length, filter_threshold, dense_offset, dense_scale):
    """start fp32 [T,768], filter_start / filter_end fp32 [T] (the document's valid rows, features in order), rows_per_feature [F]
    -> (start int8 [K,768], f2o_start int64 [K], start2end int32 [K,L])."""
    fs, fe = np.asarray(filter_start, np.float32), np.asarray(filter_end, np.float32)
    T, L = len(fs), int(max_answer_length)
    s_set, e_set = fs > filter_threshold, fe > filter_threshold          # float32 array vs Python float: compared in float32
    keep = np.flatnonzero(s_set | e_set)
    if len(keep) == 0:
        keep = np.flatnonzero(fs > -999999)[:1]
        e_set = np.zeros(T, bool)
        e_set[keep] = True
    short = np.full(T + 1, -1, np.int64)                                  # long row -> short index (end rows only); T -> -1
    short[keep[e_set[keep]]] = np.flatnonzero(e_set[keep])
    bounds = np.concatenate([[0], np.cumsum(np.asarray(rows_per_feature, np.int64))])
    hi = np.repeat(bounds[1:], np.diff(bounds))                           # each row's feature end (exclusive)
    j = keep[:, None] + np.arange(L)[None, :]
    j = np.where(j < hi[keep][:, None], j, T)
    x = (np.asarray(start, np.float32)[keep] - dense_offset) * dense_scale
    q = np.round(x.clip(-128, 127)).astype(np.int8)
    return q, keep.astype(np.int64), short[j].astype(np.int32)
