"""Benchmark of build_phrase_index.py over a phrase dump on the GPU (DESIGN.md 3.8): a seeded synthetic int8 dump written by
artifacts.write_hdf5 (several files), then run_index --stage all at IVF4096 with the draft target's sample ratios (0.2 / 0.2),
then one sub-index per half of the files (--dump_paths, --offset) and --stage merge.  Reports each stage's time, the add's rows
per second, the bytes sent to the device, and an A/B of add_int8 against add_with_ids of the same rows dequantised on the host
(same files, page cache warm, passes alternated).  The card's name and power limit are read in the same run.

    python tools/bench_index_vecs.py [--rows 4000000] [--files 8] [--rows_per_doc 100] [--ab_rows 1000000] [--ab_passes 2]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        return f'unknown ({e})'


def write_dump(dump_dir, rows, files, rows_per_doc, seed):
    from densephrases_b200 import artifacts
    os.makedirs(os.path.join(dump_dir, 'phrase'))
    rng = np.random.default_rng(seed)
    per_file = rows // files
    doc = 0
    for f in range(files):
        tree, attrs = {}, {}
        q = rng.integers(-128, 128, (per_file, 768), dtype=np.int8)
        for s in range(0, per_file, rows_per_doc):
            n = min(rows_per_doc, per_file - s)
            ntok = n + 10
            tree[str(doc)] = {'start': q[s:s + n], 'len_per_para': np.array([ntok], np.int32),
                              'f2o_start': np.arange(n, dtype=np.int32), 'word2char_start': np.arange(ntok, dtype=np.int32),
                              'word2char_end': np.arange(1, ntok + 1, dtype=np.int32)}
            attrs[str(doc)] = {'context': 'x' * ntok, 'title': str(doc), 'offset': -2.0, 'scale': 20.0}
            doc += 1
        artifacts.write_hdf5(os.path.join(dump_dir, 'phrase', f'{f}.hdf5'), tree, attrs=attrs)
    return sorted(os.path.join(dump_dir, 'phrase', n) for n in os.listdir(os.path.join(dump_dir, 'phrase')))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=4000000)
    ap.add_argument('--files', type=int, default=8)
    ap.add_argument('--rows_per_doc', type=int, default=100)
    ap.add_argument('--num_clusters', type=int, default=4096)
    ap.add_argument('--ab_rows', type=int, default=1000000)
    ap.add_argument('--ab_passes', type=int, default=2)
    ap.add_argument('--seed', type=int, default=7)
    a = ap.parse_args()
    import torch
    from densephrases_b200 import artifacts, build_index, dump
    from densephrases_b200.ivfpq import IvfPqIndex
    out = {'card': card(), 'rows': a.rows, 'files': a.files, 'rows_per_doc': a.rows_per_doc, 'num_clusters': a.num_clusters}
    tmp = tempfile.mkdtemp(prefix='bench_index_vecs_')
    try:
        d = os.path.join(tmp, 'dump')
        t0 = time.perf_counter()
        paths = write_dump(d, a.rows, a.files, a.rows_per_doc, a.seed)
        out['write_dump_s'] = time.perf_counter() - t0
        common = ['--dump_dir', d, '--fine_quant', 'OPQ96', '--num_clusters', str(a.num_clusters)]
        args = build_index.get_args(common + ['--stage', 'all'])
        t0 = time.perf_counter()
        tm = build_index.run_index(args)
        tm['total'] = time.perf_counter() - t0
        tm['add_rows_per_s'] = tm['rows'] / tm['add']
        out['all'] = tm
        half = len(paths) // 2
        subs = {}
        for off, part in ((0, paths[:half]), (10 ** 9, paths[half:])):
            sa = build_index.get_args(common + ['--stage', 'add', '--offset', str(off), '--dump_paths', ','.join(os.path.basename(p) for p in part)])
            t0 = time.perf_counter()
            st = build_index.run_index(sa)
            st['total'] = time.perf_counter() - t0
            subs[str(off)] = st
        out['sub_add'] = subs
        ma = build_index.get_args(common + ['--stage', 'merge', '--replace', '--inv_path', 'merged.ivfdata'])
        out['merge'] = build_index.run_index(ma)
        merged, single = artifacts.read_faiss_index(ma.index_path), artifacts.read_faiss_index(args.index_path)
        out['merge_lists_equal_single'] = bool(np.array_equal(merged['list_len'], single['list_len']) and
                                               np.array_equal(merged['codes'], single['codes']))
        # A/B: the same rows, read once (page cache warm), added by add_int8 from page-locked int8 and by add_with_ids from host fp32
        groups = dump.read_dump(paths[0])
        q = np.concatenate([groups[k][0]['start'] for k in sorted(groups, key=lambda s: s.encode())])[:a.ab_rows]
        pinned = build_index.pinned_rows(len(q))
        pinned[:] = q
        t = artifacts.read_faiss_index(args.trained_index_path)
        ab = {'int8': [], 'fp32': [], 'n': len(q), 'int8_h2d_bytes': q.size, 'fp32_h2d_bytes': 4 * q.size, 'fp32_host_dequant_s': []}
        for p in range(a.ab_passes):
            for kind in (('int8', 'fp32') if p % 2 == 0 else ('fp32', 'int8')):
                ix = IvfPqIndex.from_arrays(t['A'], t['centroids'], t['pq'], np.zeros(a.num_clusters, np.int64), np.zeros((0, 96), np.uint8))
                torch.cuda.synchronize()
                if kind == 'int8':
                    t0 = time.perf_counter()
                    ix.add_int8(pinned, None, -2.0, 20.0)
                    ab['int8'].append(time.perf_counter() - t0)
                else:
                    t0 = time.perf_counter()
                    x = build_index.int8_to_float(q, -2.0, 20.0)
                    t1 = time.perf_counter()
                    ix.add_with_ids(x, None)
                    ab['fp32'].append(time.perf_counter() - t1)
                    ab['fp32_host_dequant_s'].append(t1 - t0)
                    del x
                if p == 0:
                    ab[f'{kind}_lists'] = ix.lists()[1]
                del ix
        ab['same_codes'] = bool(np.array_equal(ab.pop('int8_lists'), ab.pop('fp32_lists')))
        out['ab'] = ab
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    out['card_after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
