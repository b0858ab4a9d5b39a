"""Seeded phrase dumps for the index builder's tests (tests/golden/make_index_vecs_golden.py, test_index_vecs_cpu.py and
test_index_vecs_gpu.py).  Each file is {doc name: (datasets, attrs)}, the layout dump.read_dump gives.

The names sort differently as strings and as numbers ("10" before "2"); document "7" has no rows; the documents have one to three
paragraphs (len_per_para, f2o_start); the int8 rows hold -128 and 127; the second file's offset and scale (-1.7, 17.3) are not
exact in fp32, and one of its documents uses the first file's (-2, 20).  The filter dumps give per-token filter_start /
filter_end."""
import os

import numpy as np

FILES = ('0-20.hdf5', '20-40.hdf5')
NAMES = (('2', '10', '1', '100', '3', '7', '11', '19'), ('21', '30', '200', '25', '22', '39', '24'))
ATTRS = (((-2.0, 20.0),) * 8, ((-1.7, 17.3),) * 3 + ((-2.0, 20.0),) + ((-1.7, 17.3),) * 3)
INDEX_FILTER = 0.5
# add_to_index runs: (name, files, offset, num_docs_per_add, first_passage, index_filter)
ADD_RUNS = (('all_1', (0, 1), 0, 1, False, -1e8), ('all_3', (0, 1), 0, 3, False, -1e8), ('all_2000', (0, 1), 0, 2000, False, -1e8),
            ('first', (0, 1), 0, 3, True, -1e8), ('filter', (0, 1), 0, 3, False, INDEX_FILTER),
            ('sub0', (0,), 0, 3, False, -1e8), ('sub1', (1,), 1000000000, 3, False, -1e8))
# sample_data runs: (name, doc_sample_ratio, vec_sample_ratio, norm_th)
SAMPLE_RUNS = (('r02', 0.2, 0.2, 999), ('r10', 1.0, 1.0, 999), ('r10_norm', 1.0, 1.0, 121.0), ('r05_08', 0.5, 0.8, 999))


def _doc(rng, name, offset, scale):
    if name == '7':
        n_par, rows = 1, 0
    else:
        n_par, rows = int(rng.integers(1, 4)), int(rng.integers(3, 40))
    lpp = rng.integers(max(rows, 1), 3 * max(rows, 1) + 5, n_par).astype(np.int32)
    ntok = int(lpp.sum())
    f2o = np.sort(rng.choice(ntok, rows, replace=False)).astype(np.int32)
    start = rng.integers(-128, 128, (rows, 768)).astype(np.int8)
    if rows:
        start[0, :4] = (-128, 127, -128, 127)
    words = ntok + 3
    w2s = np.sort(rng.integers(0, 5 * words, words)).astype(np.int32)
    w2e = (w2s + rng.integers(1, 5, words)).astype(np.int32)
    context = ' '.join(f'w{name}x{i}' for i in range(words))
    ds = {'start': start, 'len_per_para': lpp, 'start2end': np.zeros((rows, 10), np.int32), 'word2char_start': w2s,
          'word2char_end': w2e, 'f2o_start': f2o}
    filt = {'filter_start': rng.standard_normal(ntok).astype(np.float32), 'filter_end': rng.standard_normal(ntok).astype(np.float32)}
    return (ds, {'context': context, 'title': f'Title {name}', 'offset': offset, 'scale': scale}), (filt, {'title': f'Title {name}'})


def dumps(seed=2029):
    """-> (phrase files, filter files): lists of {doc name: (datasets, attrs)}, one per FILES entry, in the order given by NAMES."""
    rng = np.random.default_rng(seed)
    phrase, filt = [], []
    for names, attrs in zip(NAMES, ATTRS):
        p, f = {}, {}
        for name, (off, scale) in zip(names, attrs):
            p[name], f[name] = _doc(rng, name, off, scale)
        phrase.append(p)
        filt.append(f)
    return phrase, filt


def write_dumps(dump_dir, seed=2029):
    """Write dumps() as dump_dir/phrase/<file> and dump_dir/filter/<file> -> the phrase paths."""
    from densephrases_b200 import artifacts
    phrase, filt = dumps(seed)
    paths = []
    for name, p, f in zip(FILES, phrase, filt):
        for sub, groups in (('phrase', p), ('filter', f)):
            os.makedirs(os.path.join(dump_dir, sub), exist_ok=True)
            artifacts.write_hdf5(os.path.join(dump_dir, sub, name), {k: g[0] for k, g in groups.items()},
                                 attrs={k: g[1] for k, g in groups.items()})
        paths.append(os.path.join(dump_dir, 'phrase', name))
    return paths
