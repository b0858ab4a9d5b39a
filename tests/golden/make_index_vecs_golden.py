"""Golden outputs of the UNMODIFIED reference index build over a phrase dump: /root/reference/build_phrase_index.py `sample_data`
(:60-93), `add_to_index` (:156-279) and `merge_indexes` (:282-338), and scripts/preprocess/compress_metadata.py `load_doc_groups` and
`compress` (:32-91) -> tests/golden/index_vecs_reference.json.gz.

The reference modules are loaded by file path, with stand-ins in the style of make_dump_golden.py:
- h5py is a dict reader (and recorder, for idx2id files) over tests/index_vecs_cases.py's dumps.  Its files yield documents in
  byte-wise name order, as h5py does.  It hands the `offset` and `scale` attributes as Python floats, not np.float64: under
  numpy 2's promotion rules a Python float is a weak scalar, so `int8.astype(float32) / scale + offset` stays fp32, which is what
  numpy 1.x (the reference's faiss-gpu 1.6.5 environment) computed from the float64 attributes by value-based casting.
- faiss is a recorder: read_index, add_with_ids (the fp32 rows and labels of every call), write_index, and merge_from's order.
- blosc is a zlib stand-in; the golden keeps the decoded metadata, not the frames.
- tqdm is the identity.  int8_to_float is the reference's embed_utils.py, loaded as make_dump_golden.py loads it.

The fp32 rows of every add are stored as SHA-256 digests to keep the fixture small.

    python tests/golden/make_index_vecs_golden.py"""
import gzip
import hashlib
import json
import os
import pickle
import sys
import tempfile
import types
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = '/root/reference'

from tests import index_vecs_cases as cases  # noqa: E402
from tests.golden import make_dump_golden as mdg  # noqa: E402

FS = {}            # path -> {group name: _Group}
ADDS = []          # (x, ids) of every add_with_ids
MERGES = []        # sub-index paths in merge_from order
WRITTEN = {}       # index path -> number of rows added before write_index


class _Group(dict):
    def __init__(self, datasets=(), attrs=None):
        super().__init__(datasets)
        self.attrs = dict(attrs or {})

    def create_dataset(self, name, data):
        self[name] = np.array(data)


class _File(object):
    def __init__(self, path, mode='r'):
        if mode == 'w':
            FS[path] = {}
        self.g = FS[path]

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def close(self):
        pass

    def keys(self):
        return sorted(self.g, key=lambda k: k.encode())

    def items(self):
        return [(k, self.g[k]) for k in self.keys()]

    def __iter__(self):
        return iter(self.keys())

    def __len__(self):
        return len(self.g)

    def __getitem__(self, k):
        return self.g[k]

    def create_group(self, k):
        self.g[k] = _Group()
        return self.g[k]


class _Index(object):
    def __init__(self, path):
        self.path, self.nlist, self.code_size, self.ntotal = path, 8, 96, 0
        self.invlists = ('invlists', path)
        self.own_invlists = True

    def add_with_ids(self, x, ids):
        ADDS.append((np.array(x), np.array(ids)))

    def make_direct_map(self):
        pass

    def set_direct_map_type(self, t):
        pass

    def replace_invlists(self, inv):
        pass


class _OnDisk(object):
    def __init__(self, nlist, code_size, path):
        pass

    def merge_from(self, data, n):
        MERGES.extend(p for _, p in data[:n])
        return n


class _PtrVector(list):
    push_back = list.append

    def data(self):
        return list(self)

    def size(self):
        return len(self)


def reference_modules():
    _, eu = mdg.reference_modules()                   # the reference's embed_utils (int8_to_float), as make_dump_golden loads it
    h5 = types.ModuleType('h5py')
    h5.File = _File
    sys.modules['h5py'] = h5
    fa = types.ModuleType('faiss')
    fa.read_index = lambda path, *flags: _Index(path)
    fa.write_index = lambda index, path: WRITTEN.__setitem__(path, len(ADDS))
    fa.extract_index_ivf = lambda index: index
    fa.DirectMap = types.SimpleNamespace(Hashtable=2)
    fa.IO_FLAG_MMAP = 1
    fa.OnDiskInvertedLists = _OnDisk
    fa.InvertedListsPtrVector = _PtrVector
    sys.modules['faiss'] = fa
    tq = types.ModuleType('tqdm')
    tq.tqdm = lambda it=None, *a, **k: it
    sys.modules['tqdm'] = tq
    bl = types.ModuleType('blosc')
    bl.compress = lambda data, typesize=8, cname='blosclz', **k: zlib.compress(bytes(data))
    bl.decompress = zlib.decompress
    sys.modules['blosc'] = bl
    dp = sys.modules['densephrases']
    dp.Options = object
    sys.modules['densephrases.utils.embed_utils'] = eu
    bpi = mdg.load('build_phrase_index', os.path.join(REF, 'build_phrase_index.py'))
    cm = mdg.load('compress_metadata', os.path.join(REF, 'scripts', 'preprocess', 'compress_metadata.py'))
    return bpi, cm


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    bpi, cm = reference_modules()
    phrase, filt = cases.dumps()
    out = {'sample': {}, 'add': {}, 'merge': {}, 'meta': {}}
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for name, p, f in zip(cases.FILES, phrase, filt):
            for sub, groups in (('phrase', p), ('filter', f)):
                path = os.path.join(tmp, 'dump', sub, name)
                FS[path] = {k: _Group(ds, {a: (float(v) if isinstance(v, float) else v) for a, v in attrs.items()})
                            for k, (ds, attrs) in groups.items()}
            paths.append(os.path.join(tmp, 'dump', 'phrase', name))
        for name, dr, vr, th in cases.SAMPLE_RUNS:
            x, avg, std = bpi.sample_data(paths, doc_sample_ratio=dr, vec_sample_ratio=vr, norm_th=th)
            out['sample'][name] = {'shape': list(x.shape), 'dtype': str(x.dtype), 'x': sha(x), 'avg_vec': sha(avg), 'std_vec': sha(std),
                                   'avg_dtype': str(avg.dtype)}
        for name, files, offset, ndpa, first, filt_th in cases.ADD_RUNS:
            del ADDS[:]
            target, idx2id = os.path.join(tmp, f'{name}.faiss'), os.path.join(tmp, f'{name}.hdf5')
            bpi.add_to_index([paths[i] for i in files], 'trained.faiss', target, idx2id, num_docs_per_add=ndpa, fine_quant='OPQ96',
                             offset=offset, first_passage=first, index_filter=filt_th)
            x = np.concatenate([a for a, _ in ADDS])
            g = FS[idx2id][str(offset)]
            out['add'][name] = {'calls': [[sha(a), len(a), str(a.dtype)] for a, _ in ADDS], 'x': sha(x), 'n': len(x),
                                'ids': np.concatenate([i for _, i in ADDS]).tolist(), 'doc': g['doc'].tolist(), 'word': g['word'].tolist(),
                                'doc_dtype': str(g['doc'].dtype), 'offset_attr': int(g.attrs['offset'])}
        sub = os.path.join(tmp, 'index')
        os.makedirs(sub)
        for name in ('sub0', 'sub1'):
            off = [r for r in cases.ADD_RUNS if r[0] == name][0][2]
            FS[os.path.join(sub, f'{off}.hdf5')] = FS[os.path.join(tmp, f'{name}.hdf5')]
            open(os.path.join(sub, f'{off}.hdf5'), 'w').close()
            open(os.path.join(sub, f'{off}.faiss'), 'w').close()
        merged = os.path.join(tmp, 'idx2id.hdf5')
        bpi.merge_indexes(sub, 'trained.faiss', os.path.join(tmp, 'index.faiss'), merged, os.path.join(tmp, 'merged.ivfdata'))
        out['merge'] = {'sources': sorted(os.path.basename(p) for p in MERGES),
                        'idx2id': {k: {'doc': g['doc'].tolist(), 'word': g['word'].tolist()} for k, g in FS[merged].items()}}
        phrase_dir = os.path.join(tmp, 'dump', 'phrase')
        cm.os = types.SimpleNamespace(listdir=lambda d: sorted(cases.FILES, reverse=True), path=os.path)
        groups = cm.compress(cm.load_doc_groups(phrase_dir))
        pickle.dumps(groups)
        meta = {}
        for key, rec in groups.items():
            meta[key] = {'keys': list(rec), 'dtypes': {k: str(v) for k, v in rec['dtypes'].items()}, 'title': rec['title'],
                         'context': zlib.decompress(rec['context']).decode('utf-8')}
            for t in ('word2char_start', 'word2char_end', 'f2o_start'):
                meta[key][t] = np.frombuffer(zlib.decompress(rec[t]), rec['dtypes'][t]).tolist()
        out['meta'] = {'order': list(groups), 'records': meta}
    path = os.path.join(ROOT, 'tests', 'golden', 'index_vecs_reference.json.gz')
    with open(path, 'wb') as f, gzip.GzipFile(fileobj=f, mode='wb', mtime=0) as z:
        z.write(json.dumps(out, separators=(',', ':')).encode())
    print('wrote', path, os.path.getsize(path), 'bytes')
    print({k: (v['n'], len(v['calls'])) for k, v in out['add'].items()})
    print({k: v['shape'] for k, v in out['sample'].items()})


if __name__ == '__main__':
    main()
