"""Readers for the reference's on-disk artefacts, without faiss / h5py / blosc (SURVEY.md 8f #2, 8a-a14).

  index.faiss          faiss.write_index output of build_phrase_index.py:142,278,338  ->  read_faiss_index()
  idx2id.hdf5          groups '<offset>' with int datasets 'doc', 'word' (:272-276,291-301) ->  read_idx2id()
  meta_compressed.pkl  pickle of {doc_idx: blosc-zlib blobs + dtypes + title} (scripts/preprocess/compress_metadata.py:32-53)
                       ->  read_meta() / blosc_decompress()

STATUS: the three formats are restated from their published specifications / upstream serialisation code as remembered
(faiss 1.6.x impl/index_write.cpp, the HDF5 File Format Specification 2.0 as written by libhdf5 1.10 with default settings,
c-blosc 1.x's frame header), because none of those libraries -- and no file produced by them -- exists in the build container.
The test-suite can therefore only check the readers against the writers in this module (tests/test_artifacts.py); the first load of
a real released index should be cross-checked once with tools/convert_reference_artifacts.py on a machine that has the libraries.
Unknown record types fail loudly (ValueError naming the fourcc / message), they are never skipped silently.

The writers (write_faiss_index, write_hdf5, blosc_compress) emit the same subset; they exist for the tests and for exporting an
index built by densephrases_b200/build_index.py in the reference's container format."""
import mmap
import os
import pickle
import struct
import zlib

import numpy as np

# =====================================================================================================================
# FAISS index file:  IxPT( LTra(A,b) , IwPQ( ivf header( IxFI quantizer, direct map ), PQ, inverted lists ilar | ilod ) )
# =====================================================================================================================


class _Cursor:
    def __init__(self, buf, pos=0):
        self.buf, self.pos = buf, pos

    def take(self, fmt):
        size = struct.calcsize(fmt)
        if self.pos + size > len(self.buf):
            raise ValueError('truncated file')
        v = struct.unpack_from(fmt, self.buf, self.pos)
        self.pos += size
        return v[0] if len(v) == 1 else v

    def fourcc(self):
        s = bytes(self.buf[self.pos:self.pos + 4]).decode('latin-1')
        self.pos += 4
        return s

    def vector(self, dtype, copy=True):
        """faiss WRITEVECTOR: size_t element count, then the elements."""
        n = self.take('<Q')
        return self.raw(dtype, n, copy)

    def raw(self, dtype, n, copy=True):
        dtype = np.dtype(dtype)
        nbytes = int(n) * dtype.itemsize
        if self.pos + nbytes > len(self.buf):
            raise ValueError('truncated file')
        a = np.frombuffer(self.buf, dtype=dtype, count=int(n), offset=self.pos)
        self.pos += nbytes
        return a.copy() if copy else a


def _index_header(c):
    """write_index_header: d int32, ntotal int64, two dummies int64, is_trained u8, metric_type int32 (+ metric_arg f32 if > 1)."""
    d = c.take('<i')
    ntotal = c.take('<q')
    c.take('<q'); c.take('<q')
    trained = c.take('<B')
    metric = c.take('<i')
    if metric > 1:
        c.take('<f')
    return dict(d=d, ntotal=ntotal, is_trained=bool(trained), metric=metric)


def _read_vector_transform(c):
    tag = c.fourcc()
    if tag not in ('LTra', 'rrot'):             # OPQMatrix is written as a plain LinearTransform
        raise ValueError(f'unsupported VectorTransform {tag!r} (expected the OPQ matrix as LTra)')
    have_bias = c.take('<B')
    A = c.vector('<f4')
    b = c.vector('<f4')
    d_in, d_out = c.take('<i'), c.take('<i')
    c.take('<B')                                # is_trained
    if A.size != d_in * d_out:
        raise ValueError('LinearTransform matrix size mismatch')
    return dict(A=A.reshape(d_out, d_in), b=b if have_bias else None, d_in=d_in, d_out=d_out)


def _read_flat(c):
    tag = c.fourcc()
    if tag not in ('IxFI', 'IxF2', 'IxFl'):
        raise ValueError(f'unsupported coarse quantizer {tag!r} (expected IndexFlat)')
    h = _index_header(c)
    xb = c.vector('<f4')
    return h, xb.reshape(-1, h['d']) if h['d'] else xb


def _read_direct_map(c):
    kind = c.take('<B')                         # DirectMap::Type: 0 NoMap, 1 Array, 2 Hashtable
    c.vector('<i8', copy=False)                 # array map: rebuilt on the device from the lists, not needed
    if kind == 2:
        n = c.take('<Q')
        c.raw('<i8', 2 * n, copy=False)         # (id, lo) pairs: idem
    elif kind > 2:
        raise ValueError(f'unknown direct map type {kind}')


def _read_invlists(c, path, ondisk_same_dir):
    tag = c.fourcc()
    if tag == 'il00':
        return None
    nlist = c.take('<Q')
    code_size = c.take('<Q')
    if tag == 'ilar':
        kind = c.fourcc()
        raw = c.vector('<u8')
        if kind == 'full':
            sizes = raw.astype(np.int64)
        elif kind == 'sprs':
            sizes = np.zeros(nlist, dtype=np.int64)
            sizes[raw[0::2].astype(np.int64)] = raw[1::2].astype(np.int64)
        else:
            raise ValueError(f'unknown ArrayInvertedLists size encoding {kind!r}')
        if sizes.size != nlist:
            raise ValueError('inverted list size table does not match nlist')
        ntot = int(sizes.sum())
        if ntot < 0 or ntot * (code_size + 8) > len(c.buf) - c.pos:
            raise ValueError('truncated file (inverted lists)')
        codes = np.empty((ntot, code_size), dtype=np.uint8)
        ids = np.empty(ntot, dtype=np.int64)
        at = 0
        for n in sizes.tolist():                 # per non-empty list: n*code_size code bytes, then n int64 ids
            if n:
                codes[at:at + n] = c.raw('u1', n * code_size, copy=False).reshape(n, code_size)
                ids[at:at + n] = c.raw('<i8', n, copy=False)
                at += n
        return sizes, codes, ids
    if tag == 'ilod':                            # OnDiskInvertedLists: table here, payload in a side file (merge_indexes, :320-335)
        lists = c.raw('<u8', 3 * c.take('<Q')).reshape(-1, 3)      # vector<List>: (size, capacity, offset) per list
        c.raw('<u8', 2 * c.take('<Q'), copy=False)                 # vector<Slot>: free (offset, capacity) ranges
        fname = bytes(c.vector('u1')).decode('utf-8', 'replace')
        c.take('<Q')                             # totsize
        if lists.shape[0] != nlist:
            raise ValueError('on-disk list table does not match nlist')
        if ondisk_same_dir:                      # faiss.IO_FLAG_ONDISK_SAME_DIR (index.py:30): look next to the index file
            fname = os.path.join(os.path.dirname(os.path.abspath(path)), os.path.basename(fname))
        if not os.path.exists(fname):
            raise FileNotFoundError(f'inverted-list payload {fname} referenced by {path} not found')
        payload = np.memmap(fname, dtype=np.uint8, mode='r')
        sizes = lists[:, 0].astype(np.int64)
        ntot = int(sizes.sum())
        if ntot < 0 or ntot * (code_size + 8) > payload.size:
            raise ValueError(f'{fname} is smaller than the lists it should hold')
        codes = np.empty((ntot, code_size), dtype=np.uint8)
        ids = np.empty(ntot, dtype=np.int64)
        at = 0
        for n, cap, off in lists.tolist():       # at offset: capacity*code_size code bytes, then capacity int64 ids
            if n:
                codes[at:at + n] = payload[off:off + n * code_size].reshape(n, code_size)
                ids[at:at + n] = payload[off + cap * code_size:off + cap * code_size + 8 * n].view('<i8')
                at += n
        return sizes, codes, ids
    raise ValueError(f'unsupported inverted lists {tag!r}')


def read_faiss_index(path, ondisk_same_dir=True):
    """index.faiss (IndexPreTransform(OPQMatrix) -> IndexIVFPQ over IndexFlatIP, build_phrase_index.py:113-116) ->
    dict(A [d_out,d_in], centroids [nlist,d], pq [M,ksub,dsub], list_len [nlist], codes [ntotal,M] list-major, ids [ntotal],
         nprobe, ntotal, by_residual, metric).  Exactly the arrays IvfPqIndex.from_arrays takes."""
    with open(path, 'rb') as f:
        buf = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
    c = _Cursor(buf)
    tag = c.fourcc()
    chain = []
    if tag == 'IxPT':
        _index_header(c)
        nt = c.take('<i')
        chain = [_read_vector_transform(c) for _ in range(nt)]
        tag = c.fourcc()
    if tag != 'IwPQ':
        raise ValueError(f'unsupported index type {tag!r} (expected IxPT -> IwPQ; the SQ4 / HNSW / flat variants are outside the hot path)')
    h = _index_header(c)
    nlist = c.take('<Q')
    nprobe = c.take('<Q')
    qh, centroids = _read_flat(c)
    _read_direct_map(c)
    by_residual = c.take('<B')
    code_size = c.take('<Q')
    pq_d, pq_M, pq_nbits = c.take('<Q'), c.take('<Q'), c.take('<Q')
    cent = c.vector('<f4')
    ksub = 1 << pq_nbits
    if pq_nbits != 8 or code_size != pq_M or cent.size != pq_d * ksub:
        raise ValueError('only 8-bit product quantizers are supported on this path')
    inv = _read_invlists(c, path, ondisk_same_dir)
    if inv is None:
        sizes, codes, ids = np.zeros(nlist, np.int64), np.zeros((0, code_size), np.uint8), np.zeros(0, np.int64)
    else:
        sizes, codes, ids = inv
    if len(chain) > 1:
        raise ValueError('more than one pre-transform in the chain')
    d = h['d']
    A = chain[0]['A'] if chain else np.eye(d, dtype=np.float32)
    if chain and chain[0]['b'] is not None and np.any(chain[0]['b'] != 0):
        raise ValueError('pre-transform with a non-zero bias is not supported (OPQMatrix has none)')
    if centroids.shape != (nlist, d):
        raise ValueError('coarse quantizer does not hold nlist centroids')
    return dict(A=np.ascontiguousarray(A, dtype=np.float32), centroids=np.ascontiguousarray(centroids, dtype=np.float32),
                pq=cent.reshape(pq_M, ksub, pq_d // pq_M).astype(np.float32), list_len=sizes, codes=codes, ids=ids,
                nprobe=int(nprobe), ntotal=int(h['ntotal']), by_residual=bool(by_residual), metric=h['metric'],
                quantizer_metric=qh['metric'])


def _w_header(out, d, ntotal, metric):
    out.append(struct.pack('<iqqqBi', d, ntotal, 1 << 20, 1 << 20, 1, metric))


def _w_vector(out, a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    out.append(struct.pack('<Q', a.size))
    out.append(a.tobytes())


def write_faiss_index(path, A, centroids, pq, list_len, codes, ids, nprobe=1, ondisk_payload=None):
    """Inverse of read_faiss_index for the same subset (METRIC_INNER_PRODUCT = 0).  ondisk_payload: file name -> write the lists as
    OnDiskInvertedLists ('ilod') with their payload in that side file, like merge_indexes does; else ArrayInvertedLists ('ilar')."""
    A = np.asarray(A, np.float32); centroids = np.asarray(centroids, np.float32); pq = np.asarray(pq, np.float32)
    list_len = np.asarray(list_len, np.int64); codes = np.asarray(codes, np.uint8); ids = np.asarray(ids, np.int64)
    d_out, d_in = A.shape
    nlist, d = centroids.shape
    M, ksub, dsub = pq.shape
    ntotal = int(list_len.sum())
    out = [b'IxPT']
    _w_header(out, d_in, ntotal, 0)
    out.append(struct.pack('<i', 1))
    out.append(b'LTra' + struct.pack('<B', 0))
    _w_vector(out, A.reshape(-1), '<f4'); _w_vector(out, np.zeros(0), '<f4')
    out.append(struct.pack('<iiB', d_in, d_out, 1))
    out.append(b'IwPQ')
    _w_header(out, d, ntotal, 0)
    out.append(struct.pack('<QQ', nlist, nprobe))
    out.append(b'IxFI')
    _w_header(out, d, nlist, 0)
    _w_vector(out, centroids.reshape(-1), '<f4')
    out.append(struct.pack('<B', 2)); _w_vector(out, np.zeros(0), '<i8'); out.append(struct.pack('<Q', 0))     # empty Hashtable direct map
    out.append(struct.pack('<BQ', 1, M))
    out.append(struct.pack('<QQQ', M * dsub, M, 8)); _w_vector(out, pq.reshape(-1), '<f4')
    starts = np.concatenate([[0], np.cumsum(list_len)])
    if ondisk_payload is None:
        out.append(b'ilar' + struct.pack('<QQ', nlist, M))
        nz = np.flatnonzero(list_len)
        if nz.size > nlist // 2:
            out.append(b'full'); _w_vector(out, list_len, '<u8')
        else:
            out.append(b'sprs'); _w_vector(out, np.stack([nz, list_len[nz]], 1).reshape(-1), '<u8')
        for l in nz.tolist():
            out.append(codes[starts[l]:starts[l + 1]].tobytes()); out.append(ids[starts[l]:starts[l + 1]].astype('<i8').tobytes())
    else:
        table, payload, off = [], [], 0
        for l in range(nlist):
            n = int(list_len[l]); cap = n + (n % 3)                      # capacity >= size, to exercise the layout
            table.append((n, cap, off))
            blob = bytearray(cap * M + cap * 8)
            blob[:n * M] = codes[starts[l]:starts[l + 1]].tobytes()
            blob[cap * M:cap * M + 8 * n] = ids[starts[l]:starts[l + 1]].astype('<i8').tobytes()
            payload.append(bytes(blob)); off += len(blob)
        with open(os.path.join(os.path.dirname(os.path.abspath(path)), os.path.basename(ondisk_payload)), 'wb') as f:
            f.write(b''.join(payload))
        out.append(b'ilod' + struct.pack('<QQ', nlist, M))
        out.append(struct.pack('<Q', nlist) + np.asarray(table, dtype='<u8').tobytes())      # vector<List>: count of structs, then 3 words each
        out.append(struct.pack('<Q', 0))                                                     # vector<Slot>: no free ranges
        name = ('/somewhere/else/' + os.path.basename(ondisk_payload)).encode()
        _w_vector(out, np.frombuffer(name, np.uint8), 'u1')
        out.append(struct.pack('<Q', off))
    with open(path, 'wb') as f:
        f.write(b''.join(out))


# =====================================================================================================================
# blosc 1.x frames (meta_compressed.pkl fields):  16-byte header | int32 bstarts[nblocks] | blocks of [int32 cbytes | stream]...
# =====================================================================================================================
_BLOSC_MAX_SPLITS, _BLOSC_MIN_BUFFERSIZE = 16, 128


def _unshuffle(block, typesize):
    n = len(block) // typesize
    if typesize <= 1 or n == 0:
        return block
    a = np.frombuffer(block, np.uint8)
    body = a[:n * typesize].reshape(typesize, n).T.reshape(-1)
    return body.tobytes() + a[n * typesize:].tobytes()


def _blosc_streams(buf, start, end, nsplits, neblock, codec):
    """Try to parse [start, end) as nsplits streams of `[int32 cbytes | payload]`; None if the layout does not fit exactly."""
    out, pos = [], start
    for _ in range(nsplits):
        if pos + 4 > end:
            return None
        cb = struct.unpack_from('<i', buf, pos)[0]
        pos += 4
        if cb < 0 or pos + cb > end:
            return None
        chunk = bytes(buf[pos:pos + cb])
        pos += cb
        if cb == neblock:
            out.append(chunk)                    # stored uncompressed
        else:
            try:
                raw = codec(chunk)
            except Exception:
                return None
            if len(raw) != neblock:
                return None
            out.append(raw)
    return b''.join(out) if pos == end else None


def blosc_decompress(frame):
    """c-blosc 1.x frame -> bytes.  Supports the memcpy and zlib codecs with byte shuffle (what the reference writes:
    blosc.compress(..., cname='zlib'), compress_metadata.py:43-46); blosclz / lz4 / snappy / zstd frames raise."""
    buf = memoryview(frame).cast('B') if not isinstance(frame, (bytes, bytearray)) else frame
    if len(buf) < 16:
        raise ValueError('not a blosc frame')
    version, _, flags, typesize = buf[0], buf[1], buf[2], buf[3]
    nbytes, blocksize, cbytes = struct.unpack_from('<III', buf, 4)
    if version != 2 or cbytes > len(buf):
        raise ValueError('unsupported or truncated blosc frame')
    if nbytes == 0:
        return b''
    if flags & 0x2:                              # memcpyed
        return bytes(buf[16:16 + nbytes])
    if flags & 0x4:
        raise ValueError('bit-shuffled blosc frames are not supported')
    comp = (flags >> 5) & 0x7
    if comp != 3:
        raise ValueError(f'blosc compressor format {comp} is not supported (only zlib = 3, the reference\'s choice)')
    typesize = typesize or 1
    nblocks = (nbytes + blocksize - 1) // blocksize
    bstarts = list(struct.unpack_from(f'<{nblocks}i', buf, 16))
    ends = sorted(bstarts) + [cbytes]
    out = []
    for i in range(nblocks):
        bsize = min(blocksize, nbytes - i * blocksize)
        leftover = bsize != blocksize
        start = bstarts[i]
        end = ends[ends.index(start) + 1]
        # a full-size block is either one stream or `typesize` streams (older c-blosc split every codec; newer ones record
        # "don't split" in flag 0x10) -- accept whichever parses exactly
        options = [1]
        if not leftover and 1 < typesize <= _BLOSC_MAX_SPLITS and bsize // typesize >= _BLOSC_MIN_BUFFERSIZE and bsize % typesize == 0:
            options = [1, typesize] if (flags & 0x10) else [typesize, 1]
        block = None
        for ns in options:
            block = _blosc_streams(buf, start, end, ns, bsize // ns, zlib.decompress)
            if block is not None:
                break
        if block is None:
            raise ValueError('corrupt blosc frame (block does not parse)')
        out.append(_unshuffle(block, typesize) if (flags & 0x1) else block)
    data = b''.join(out)
    if len(data) != nbytes:
        raise ValueError('corrupt blosc frame (size mismatch)')
    return data


def blosc_compress(data, typesize=8, shuffle=True, blocksize=None, split=False, clevel=6):
    """Writer for the same subset (zlib codec, optional byte shuffle / split streams / memcpy for tiny inputs)."""
    data = bytes(data)
    nbytes = len(data)
    if nbytes < 128:                             # c-blosc stores tiny buffers uncompressed
        return struct.pack('<BBBBIII', 2, 1, 0x2 | (0x1 if shuffle else 0), typesize, nbytes, nbytes, nbytes + 16) + data
    blocksize = blocksize or max(typesize * 128, 1 << 15)
    blocksize = min(blocksize - blocksize % typesize or typesize, nbytes)
    nblocks = (nbytes + blocksize - 1) // blocksize
    blocks = []
    for i in range(nblocks):
        raw = data[i * blocksize:(i + 1) * blocksize]
        if shuffle and typesize > 1:
            n = len(raw) // typesize
            a = np.frombuffer(raw, np.uint8)
            raw = a[:n * typesize].reshape(n, typesize).T.reshape(-1).tobytes() + a[n * typesize:].tobytes()
        full = len(raw) == blocksize
        ns = typesize if (split and full and 1 < typesize <= _BLOSC_MAX_SPLITS and blocksize // typesize >= _BLOSC_MIN_BUFFERSIZE
                          and blocksize % typesize == 0) else 1
        ne = len(raw) // ns
        parts = []
        for s in range(ns):
            piece = raw[s * ne:(s + 1) * ne]
            z = zlib.compress(piece, clevel)
            if len(z) >= len(piece):
                z = piece
            parts.append(struct.pack('<i', len(z)) + z)
        blocks.append(b''.join(parts))
    flags = (3 << 5) | (0x1 if shuffle else 0) | (0 if split else 0x10)
    bstarts, off = [], 16 + 4 * nblocks
    for b in blocks:
        bstarts.append(off); off += len(b)
    return struct.pack('<BBBBIII', 2, 1, flags, typesize, nbytes, blocksize, off) + struct.pack(f'<{nblocks}i', *bstarts) + b''.join(blocks)


def read_meta(path):
    """meta_compressed.pkl -> {doc_idx: record} with blosc blobs decoded lazily by MIPS.decompress_meta (index.py:106-122)."""
    with open(path, 'rb') as f:
        return pickle.load(f)


def compress_meta(doc_groups):
    """compress_metadata.py:compress (:32-70) of {doc_idx: {word2char_start, word2char_end, f2o_start, context, title}}, in place:
    the three arrays as blosc-zlib frames of typesize 1, the context as a blosc-zlib frame of its UTF-8 bytes (python-blosc's
    defaults: typesize 8, byte shuffle, level 9), the arrays' dtypes under 'dtypes', the title as it is.  The frames decode to the
    same bytes as c-blosc's; the bytes of the frames themselves may differ."""
    for rec in doc_groups.values():
        dtypes = {name: rec[name].dtype for name in ('word2char_start', 'word2char_end', 'f2o_start')}
        for name in dtypes:
            rec[name] = blosc_compress(np.ascontiguousarray(rec[name]).tobytes(), typesize=1, clevel=9)
        rec['context'] = blosc_compress(rec['context'].encode('utf-8'), typesize=8, clevel=9)
        rec['dtypes'] = dtypes
    return doc_groups


def write_meta(input_dump_dir, output_dir):
    """scripts/preprocess/compress_metadata.py (:72-111): the metadata of every `*hdf5*` file of input_dump_dir (sorted; a document in
    several files keeps its first position and its last record), compressed by compress_meta, pickled to
    output_dir/meta_compressed.pkl, which MIPS reads.  -> the output path."""
    doc_groups = {}
    for name in sorted(n for n in os.listdir(input_dump_dir) if 'hdf5' in n):
        h = open_hdf5(os.path.join(input_dump_dir, name))
        for key, addr in h.children(h.root_addr).items():
            members, attrs = h.children(addr), h.attributes(addr)
            rec = {t: h.dataset(members[t]) for t in ('word2char_start', 'word2char_end', 'f2o_start')}
            rec['context'], rec['title'] = attrs['context'], attrs['title']
            doc_groups[key] = rec
    out = os.path.join(output_dir, 'meta_compressed.pkl')
    with open(out, 'wb') as f:
        pickle.dump(compress_meta(doc_groups), f)
    return out


def decode_meta_field(value, dtype=None):
    """A metadata field as stored by the reference (blosc frame), by this repo's converter (zlib stream) or raw."""
    if isinstance(value, (bytes, bytearray, memoryview)):
        b = bytes(value)
        if len(b) >= 16 and b[0] == 2 and struct.unpack_from('<I', b, 12)[0] == len(b):
            raw = blosc_decompress(b)
        else:
            raw = zlib.decompress(b)
        return np.frombuffer(raw, dtype) if dtype is not None else raw
    return np.asarray(value) if dtype is not None else value


# =====================================================================================================================
# HDF5 (the subset h5py writes with default settings: superblock v0/v1, version-1 object headers, symbol-table groups = v1 B-tree +
# local heap + SNOD nodes, contiguous / compact / chunked(+deflate, shuffle) datasets of little- or big-endian integers and floats)
# =====================================================================================================================
_H5_SIG = b'\x89HDF\r\n\x1a\n'
_UNDEF = 0xFFFFFFFFFFFFFFFF


class _H5:
    def __init__(self, buf):
        self.buf = buf
        base = 0
        while bytes(buf[base:base + 8]) != _H5_SIG:          # the superblock may sit behind a user block at 512, 1024, ...
            base = 512 if base == 0 else base * 2
            if base + 8 > len(buf):
                raise ValueError('not an HDF5 file')
        ver = buf[base + 8]
        if ver > 1:
            raise ValueError(f'HDF5 superblock version {ver} (libver="latest" files) is not supported; h5py writes version 0 by default')
        if buf[base + 13] != 8 or buf[base + 14] != 8:
            raise ValueError('only 8-byte offsets / lengths are supported')
        pos = base + 24 + (4 if ver == 1 else 0)
        self.base = struct.unpack_from('<Q', buf, pos)[0]
        root_entry = pos + 32                                  # base, free-space, eof, driver-info addresses, then the root symbol table entry
        self.root_header = struct.unpack_from('<Q', buf, root_entry + 8)[0]

    def u(self, fmt, addr):
        return struct.unpack_from(fmt, self.buf, self.base + addr)

    # -- object headers ------------------------------------------------------------------------------------------------
    def messages(self, addr):
        """Version-1 object header at addr -> [(type, flags, absolute data offset, size)] across continuation blocks."""
        a = self.base + addr
        if bytes(self.buf[a:a + 4]) == b'OHDR':
            raise ValueError('version-2 object headers (libver="latest") are not supported')
        version, _, nmsg, _, hsize = struct.unpack_from('<BBHII', self.buf, a)
        if version != 1:
            raise ValueError(f'object header version {version} not supported')
        blocks = [(a + 16, hsize)]
        out = []
        while blocks and len(out) < nmsg:
            pos, left = blocks.pop(0)
            end = pos + left
            while pos + 8 <= end and len(out) < nmsg:
                mtype, msize, mflags = struct.unpack_from('<HHB', self.buf, pos)
                data = pos + 8
                out.append((mtype, mflags, data, msize))
                if mtype == 0x0010:                            # continuation: (offset, length)
                    off, length = struct.unpack_from('<QQ', self.buf, data)
                    blocks.append((self.base + off, length))
                pos = data + msize
        return out

    # -- groups ---------------------------------------------------------------------------------------------------------
    def _heap_name(self, heap_addr, off):
        a = self.base + heap_addr
        if bytes(self.buf[a:a + 4]) != b'HEAP':
            raise ValueError('bad local heap signature')
        data_addr = struct.unpack_from('<Q', self.buf, a + 24)[0]
        s = self.base + data_addr + off
        e = s
        while self.buf[e] != 0:
            e += 1
        return bytes(self.buf[s:e]).decode('utf-8')

    def _walk_group_tree(self, node_addr, heap_addr, out):
        a = self.base + node_addr
        if bytes(self.buf[a:a + 4]) != b'TREE':
            raise ValueError('bad B-tree node signature')
        ntype, level, used = struct.unpack_from('<BBH', self.buf, a + 4)
        if ntype != 0:
            raise ValueError('expected a group B-tree node')
        pos = a + 24 + 8                                      # skip siblings and key 0
        for _ in range(used):
            child = struct.unpack_from('<Q', self.buf, pos)[0]
            pos += 16                                          # child + next key
            if level > 0:
                self._walk_group_tree(child, heap_addr, out)
                continue
            s = self.base + child
            if bytes(self.buf[s:s + 4]) != b'SNOD':
                raise ValueError('bad symbol node signature')
            nsym = struct.unpack_from('<H', self.buf, s + 6)[0]
            for i in range(nsym):
                name_off, header = struct.unpack_from('<QQ', self.buf, s + 8 + 40 * i)
                out[self._heap_name(heap_addr, name_off)] = header

    def children(self, addr):
        """object header address -> {name: object header address} if it is a (symbol-table) group, else None."""
        for mtype, _, data, _ in self.messages(addr):
            if mtype == 0x0011:
                btree, heap = struct.unpack_from('<QQ', self.buf, data)
                out = {}
                self._walk_group_tree(btree, heap, out)
                return out
            if mtype in (0x0002, 0x0006):
                raise ValueError('new-style (link message) groups are not supported')
        return None

    # -- attributes (object-header attribute messages; h5py's default for small attributes) ---------------------------------
    @property
    def root_addr(self):
        return self.root_header

    def _global_heap_object(self, coll_addr, index):
        a = self.base + coll_addr
        if bytes(self.buf[a:a + 4]) != b'GCOL':
            raise ValueError('bad global heap collection signature')
        size = struct.unpack_from('<Q', self.buf, a + 8)[0]
        pos, end = a + 16, a + size
        while pos + 16 <= end:
            idx, _, _, osize = struct.unpack_from('<HHIQ', self.buf, pos)
            if idx == 0:
                break
            if idx == index:
                return bytes(self.buf[pos + 16:pos + 16 + osize])
            pos += 16 + ((osize + 7) // 8) * 8
        raise ValueError(f'global heap object {index} not found')

    def _attr_value(self, dt_at, ds_at, data_at):
        cls_ver, b0, b1, _, size = struct.unpack_from('<BBBBI', self.buf, dt_at)
        cls = cls_ver & 0x0F
        sver, rank = struct.unpack_from('<BB', self.buf, ds_at)
        dims = struct.unpack_from(f'<{rank}Q', self.buf, ds_at + (8 if sver == 1 else 4)) if rank else ()
        count = int(np.prod(dims)) if rank else 1
        if cls == 3:                                            # fixed-length string (null-terminated / null- or space-padded)
            vals = [bytes(self.buf[data_at + i * size:data_at + (i + 1) * size]).split(b'\0')[0].decode('utf-8') for i in range(count)]
        elif cls == 9 and (b0 & 0x0F) == 1:                     # variable-length string: (length, global heap collection, index)
            vals = []
            for i in range(count):
                n, coll, idx = struct.unpack_from('<IQI', self.buf, data_at + 16 * i)
                vals.append(self._global_heap_object(coll, idx)[:n].decode('utf-8') if n else '')
        elif cls in (0, 1):
            vals = np.frombuffer(self.buf, self._dtype(dt_at), count, data_at).copy()
            return vals.reshape(dims) if rank else vals[0]
        else:
            raise ValueError(f'attribute datatype class {cls} is not supported')
        return vals[0] if not rank else vals

    def attributes(self, addr):
        """object header address -> {attribute name: str | number | ndarray} (attribute message versions 1-3)."""
        out = {}
        for mtype, _, data, msize in self.messages(addr):
            if mtype != 0x000C:
                continue
            ver = self.buf[data]
            name_sz, dt_sz, ds_sz = struct.unpack_from('<HHH', self.buf, data + 2)
            if ver == 1:
                pad = lambda n: (n + 7) // 8 * 8
                pos = data + 8
            elif ver in (2, 3):
                if self.buf[data + 1] & 0x03:
                    raise ValueError('shared attribute datatypes / dataspaces are not supported')
                pad = lambda n: n
                pos = data + (9 if ver == 3 else 8)
            else:
                raise ValueError(f'attribute message version {ver} not supported')
            name = bytes(self.buf[pos:pos + name_sz]).split(b'\0')[0].decode('utf-8')
            dt_at = pos + pad(name_sz)
            ds_at = dt_at + pad(dt_sz)
            out[name] = self._attr_value(dt_at, ds_at, ds_at + pad(ds_sz))
        return out

    # -- datasets -------------------------------------------------------------------------------------------------------
    def _dtype(self, data):
        cls_ver, b0, _, _, size = struct.unpack_from('<BBBBI', self.buf, data)
        cls = cls_ver & 0x0F
        order = '>' if (b0 & 1) else '<'
        if cls == 0:
            return np.dtype(f"{order}{'i' if (b0 & 0x08) else 'u'}{size}")
        if cls == 1:
            return np.dtype(f'{order}f{size}')
        raise ValueError(f'HDF5 datatype class {cls} is not supported (integers and floats only)')

    def _filters(self, data):
        version, n = struct.unpack_from('<BB', self.buf, data)
        if version != 1:
            raise ValueError('filter pipeline version 2 not supported')
        pos, out = data + 8, []
        for _ in range(n):
            fid, nlen, _, ncd = struct.unpack_from('<HHHH', self.buf, pos)
            pos += 8 + ((nlen + 7) // 8) * 8 + 4 * (ncd + (ncd & 1))
            out.append(fid)
        return out

    def dataset(self, addr):
        shape = dtype = layout = None
        filters = []
        for mtype, _, data, size in self.messages(addr):
            if mtype == 0x0001:
                ver, rank, flags = struct.unpack_from('<BBB', self.buf, data)
                dims_at = data + (8 if ver == 1 else 4)
                shape = struct.unpack_from(f'<{rank}Q', self.buf, dims_at)
            elif mtype == 0x0003:
                dtype = self._dtype(data)
            elif mtype == 0x000B:
                filters = self._filters(data)
            elif mtype == 0x0008:
                layout = data
        if shape is None or dtype is None or layout is None:
            raise ValueError('object is not a dataset (dataspace / datatype / layout message missing)')
        count = int(np.prod(shape)) if len(shape) else 1
        ver, cls = struct.unpack_from('<BB', self.buf, layout)
        if ver != 3:
            raise ValueError(f'data layout message version {ver} not supported')
        if cls == 0:                                            # compact
            n = struct.unpack_from('<H', self.buf, layout + 2)[0]
            raw = bytes(self.buf[layout + 4:layout + 4 + n])
            return np.frombuffer(raw, dtype, count).reshape(shape).copy()
        if cls == 1:                                            # contiguous
            a, n = struct.unpack_from('<QQ', self.buf, layout + 2)
            if a == _UNDEF:
                return np.zeros(shape, dtype)
            return np.frombuffer(self.buf, dtype, count, self.base + a).reshape(shape).copy()
        if cls == 2:                                            # chunked, version-1 B-tree index
            ndim1 = self.buf[layout + 2]
            btree = struct.unpack_from('<Q', self.buf, layout + 3)[0]
            cdims = struct.unpack_from(f'<{ndim1}I', self.buf, layout + 11)[:-1]
            out = np.zeros(shape, dtype)
            if btree != _UNDEF:
                self._walk_chunks(btree, ndim1, cdims, filters, dtype, out)
            return out
        raise ValueError(f'data layout class {cls} not supported')

    def _walk_chunks(self, node_addr, ndim1, cdims, filters, dtype, out):
        a = self.base + node_addr
        if bytes(self.buf[a:a + 4]) != b'TREE':
            raise ValueError('bad chunk B-tree signature')
        ntype, level, used = struct.unpack_from('<BBH', self.buf, a + 4)
        if ntype != 1:
            raise ValueError('expected a chunk B-tree node')
        ksize = 8 + 8 * ndim1
        pos = a + 24
        for _ in range(used):
            csize, fmask = struct.unpack_from('<II', self.buf, pos)
            offs = struct.unpack_from(f'<{ndim1}Q', self.buf, pos + 8)[:-1]
            child = struct.unpack_from('<Q', self.buf, pos + ksize)[0]
            pos += ksize + 8
            if level > 0:
                self._walk_chunks(child, ndim1, cdims, filters, dtype, out)
                continue
            raw = bytes(self.buf[self.base + child:self.base + child + csize])
            for k, fid in reversed(list(enumerate(filters))):
                if fmask & (1 << k):
                    continue
                if fid == 1:
                    raw = zlib.decompress(raw)
                elif fid == 2:
                    raw = _unshuffle(raw, dtype.itemsize)
                elif fid == 3:
                    raw = raw[:-4]                              # fletcher32 checksum, not verified
                else:
                    raise ValueError(f'HDF5 filter {fid} not supported')
            chunk = np.frombuffer(raw, dtype, int(np.prod(cdims))).reshape(cdims)
            sel = tuple(slice(o, min(o + c, s)) for o, c, s in zip(offs, cdims, out.shape))
            out[sel] = chunk[tuple(slice(0, s.stop - s.start) for s in sel)]


def read_hdf5(path, max_depth=8):
    """-> nested dict {name: dict (group) | ndarray (dataset)} of the whole file (meant for small tables like idx2id.hdf5)."""
    with open(path, 'rb') as f:
        buf = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)

    def visit(h, addr, depth):
        kids = h.children(addr)
        if kids is None:
            return h.dataset(addr)
        if depth > max_depth:
            raise ValueError('group nesting too deep')
        return {name: visit(h, a, depth + 1) for name, a in kids.items()}

    try:
        h = _H5(buf)
        return visit(h, h.root_header, 0)
    except (struct.error, IndexError, OverflowError, UnicodeDecodeError, TypeError, RecursionError, MemoryError) as e:
        raise ValueError(f'corrupt or unsupported HDF5 file {path}: {type(e).__name__}: {e}') from e


def open_hdf5(path):
    """-> the lazy reader (`children(addr)`, `dataset(addr)`, `attributes(addr)`, `root_addr`) over a memory map of the file."""
    with open(path, 'rb') as f:
        buf = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ)
    return _H5(buf)


def read_idx2id(path):
    """idx2id.hdf5 -> {offset_key: {'doc': ints, 'word': ints}} (MIPS.load_idx_f, index.py:78-88)."""
    tree = read_hdf5(path)
    return {key: {t: np.asarray(g[t]) for t in ('doc', 'word')} for key, g in tree.items()}


class _H5Writer:
    """Emits the same subset: superblock v0, version-1 object headers, group B-trees of as many levels as the links need,
    contiguous datasets.  Test / export helper."""
    LEAF_K, INTERNAL_K = 4, 16

    def __init__(self):
        self.b = bytearray(96)

    def alloc(self, data):
        while len(self.b) % 8:
            self.b.append(0)
        at = len(self.b)
        self.b += data
        return at

    @staticmethod
    def _msg(mtype, data):
        data = bytes(data) + b'\0' * (-len(data) % 8)
        return struct.pack('<HHBBBB', mtype, len(data), 0, 0, 0, 0) + data

    def _header(self, msgs):
        body = b''.join(msgs)
        return self.alloc(struct.pack('<BBHII', 1, 0, len(msgs), 1, len(body)) + b'\0' * 4 + body)

    def dataset(self, arr):
        arr = np.ascontiguousarray(arr)
        dt = arr.dtype
        if dt.kind in 'iu':
            tmsg = struct.pack('<BBBBI', 0x10, (1 if dt.byteorder == '>' else 0) | (0x08 if dt.kind == 'i' else 0), 0, 0, dt.itemsize) + \
                struct.pack('<HH', 0, 8 * dt.itemsize)
        elif dt.kind == 'f' and dt.itemsize in (4, 8):
            sign = 31 if dt.itemsize == 4 else 63
            prop = struct.pack('<HHBBBBI', 0, 8 * dt.itemsize, 23, 8, 0, 23, 127) if dt.itemsize == 4 else struct.pack('<HHBBBBI', 0, 64, 52, 11, 0, 52, 1023)
            tmsg = struct.pack('<BBBBI', 0x11, 0x20 | (1 if dt.byteorder == '>' else 0), sign, 0, dt.itemsize) + prop
        else:
            raise ValueError(f'dtype {dt} not supported by the HDF5 writer')
        data_at = self.alloc(arr.tobytes()) if arr.size else _UNDEF
        space = struct.pack('<BBBBI', 1, arr.ndim, 0, 0, 0) + struct.pack(f'<{arr.ndim}Q', *arr.shape)
        layout = struct.pack('<BBQQ', 3, 1, data_at, arr.nbytes)
        return self._header([self._msg(0x0001, space), self._msg(0x0003, tmsg), self._msg(0x0008, layout)])

    def dataset_chunked(self, arr, chunks, deflate=True, shuffle=True):
        """Chunked layout with a one-node version-1 chunk B-tree (<= 64 chunks), optional shuffle + deflate filters."""
        arr = np.ascontiguousarray(arr)
        dt = arr.dtype
        if dt.kind not in 'iu':
            raise ValueError('chunked writer: integer dtypes only')
        grid = [range(0, s, c) for s, c in zip(arr.shape, chunks)]
        keys = []
        for offs in np.stack(np.meshgrid(*grid, indexing='ij'), -1).reshape(-1, arr.ndim).tolist():
            block = np.zeros(chunks, dt)
            sel = tuple(slice(o, min(o + c, s)) for o, c, s in zip(offs, chunks, arr.shape))
            block[tuple(slice(0, s.stop - s.start) for s in sel)] = arr[sel]
            raw = block.tobytes()
            if shuffle and dt.itemsize > 1:
                n = len(raw) // dt.itemsize
                raw = np.frombuffer(raw, np.uint8).reshape(n, dt.itemsize).T.reshape(-1).tobytes()
            if deflate:
                raw = zlib.compress(raw, 4)
            keys.append((len(raw), offs, self.alloc(raw)))
        if len(keys) > 64:
            raise ValueError('too many chunks for the one-node chunk writer')
        node = b'TREE' + struct.pack('<BBHQQ', 1, 0, len(keys), _UNDEF, _UNDEF)
        for size, offs, at in keys:
            node += struct.pack('<II', size, 0) + struct.pack(f'<{arr.ndim + 1}Q', *offs, 0) + struct.pack('<Q', at)
        node += struct.pack('<II', 0, 0) + struct.pack(f'<{arr.ndim + 1}Q', *arr.shape, 0)
        tree_at = self.alloc(node)
        tmsg = struct.pack('<BBBBI', 0x10, (1 if dt.byteorder == '>' else 0) | (0x08 if dt.kind == 'i' else 0), 0, 0, dt.itemsize) + \
            struct.pack('<HH', 0, 8 * dt.itemsize)
        space = struct.pack('<BBBBI', 1, arr.ndim, 0, 0, 0) + struct.pack(f'<{arr.ndim}Q', *arr.shape)
        layout = struct.pack('<BBB', 3, 2, arr.ndim + 1) + struct.pack('<Q', tree_at) + struct.pack(f'<{arr.ndim + 1}I', *chunks, dt.itemsize)
        filt = []
        if shuffle and dt.itemsize > 1:
            filt.append(struct.pack('<HHHH', 2, 0, 1, 1) + struct.pack('<II', dt.itemsize, 0))
        if deflate:
            filt.append(struct.pack('<HHHH', 1, 0, 1, 1) + struct.pack('<II', 4, 0))
        msgs = [self._msg(0x0001, space), self._msg(0x0003, tmsg)]
        if filt:
            msgs.append(self._msg(0x000B, struct.pack('<BBHI', 1, len(filt), 0, 0) + b''.join(filt)))
        msgs.append(self._msg(0x0008, layout))
        return self._header(msgs)

    def _attr_msgs(self, attrs):
        """{name: str (variable-length UTF-8 string in a global heap collection, what h5py writes for `g.attrs[k] = "text"`) |
        bytes (fixed-length string) | float (float64 scalar) | int (int64 scalar)} -> version-1 attribute messages."""
        if not attrs:
            return []
        vlen = [(k, v.encode('utf-8')) for k, v in attrs.items() if isinstance(v, str)]
        objs, coll_at = {}, 0
        if vlen:
            body = bytearray()
            for i, (k, raw) in enumerate(vlen, 1):
                objs[k] = (i, len(raw))
                body += struct.pack('<HHIQ', i, 1, 0, len(raw)) + raw + b'\0' * (-len(raw) % 8)
            total = max(4096, 16 + len(body) + 16)
            free = total - 16 - len(body)
            body += struct.pack('<HHIQ', 0, 0, 0, free) + b'\0' * (free - 16)
            coll_at = self.alloc(b'GCOL' + struct.pack('<BBBBQ', 1, 0, 0, 0, total) + bytes(body))
        msgs = []
        space = struct.pack('<BBBBI', 1, 0, 0, 0, 0)                                       # scalar dataspace
        for k, v in attrs.items():
            name = k.encode('utf-8') + b'\0'
            if isinstance(v, str):
                dt = struct.pack('<BBBBI', 0x19, 0x01, 0x01, 0, 16) + struct.pack('<BBBBI', 0x13, 0x10, 0, 0, 1)   # vlen string of UTF-8 chars
                idx, n = objs[k]
                data = struct.pack('<IQI', n, coll_at, idx)
            elif isinstance(v, float):                                                     # what h5py writes for a Python float
                dt = struct.pack('<BBBBI', 0x11, 0x20, 63, 0, 8) + struct.pack('<HHBBBBI', 0, 64, 52, 11, 0, 52, 1023)
                data = struct.pack('<d', v)
            elif isinstance(v, int) and not isinstance(v, bool):                           # ... and for a Python int
                dt = struct.pack('<BBBBI', 0x10, 0x08, 0, 0, 8) + struct.pack('<HH', 0, 64)
                data = struct.pack('<q', v)
            else:
                raw = bytes(v) + b'\0'
                dt = struct.pack('<BBBBI', 0x13, 0x00, 0, 0, len(raw))                      # null-terminated ASCII string
                data = raw
            p8 = lambda b: b + b'\0' * (-len(b) % 8)
            msgs.append(self._msg(0x000C, struct.pack('<BBHHH', 1, 0, len(name), len(dt), len(space)) + p8(name) + p8(dt) + p8(space) + data))
        return msgs

    def group(self, links, attrs=None):
        """links {name: object header address} -> (header address, btree address, heap address)"""
        names = sorted(links)                                  # the B-tree orders links by name
        heap = bytearray(8)                                    # offset 0: the empty name
        offs = {}
        for n in names:
            offs[n] = len(heap)
            e = n.encode('utf-8') + b'\0'
            heap += e + b'\0' * (-len(e) % 8)
        heap_data = self.alloc(bytes(heap))
        heap_at = self.alloc(b'HEAP' + struct.pack('<BBBBQQQ', 0, 0, 0, 0, len(heap), _UNDEF, heap_data))
        per = 2 * self.LEAF_K
        snods, keys = [], [0]
        for i in range(0, len(names), per):
            part = names[i:i + per]
            ent = b''.join(struct.pack('<QQII', offs[n], links[n], 0, 0) + b'\0' * 16 for n in part)
            ent += b'\0' * (40 * (per - len(part)))
            snods.append(self.alloc(b'SNOD' + struct.pack('<BBH', 1, 0, len(part)) + ent))
            keys.append(offs[part[-1]])
        # B-tree levels bottom up, at most 2 * INTERNAL_K children per node; the nodes of a level are linked to their left and right
        # siblings (libhdf5 may walk a level through them).  Up to 256 links this is the single level-0 node written before.
        fan, level, children = 2 * self.INTERNAL_K, 0, snods
        while True:
            parts = [(children[i:i + fan], keys[i:i + fan + 1]) for i in range(0, len(children), fan)]
            nodes = [self._tree_node(level, c, k) for c, k in parts]
            for left, right in zip(nodes, nodes[1:]):
                struct.pack_into('<Q', self.b, left + 16, right)
                struct.pack_into('<Q', self.b, right + 8, left)
            if len(nodes) == 1:
                tree_at = nodes[0]
                break
            keys = [k[0] for _, k in parts] + [parts[-1][1][-1]]
            children, level = nodes, level + 1
        return self._header([self._msg(0x0011, struct.pack('<QQ', tree_at, heap_at))] + self._attr_msgs(attrs)), tree_at, heap_at

    def _tree_node(self, level, children, keys):
        node = b'TREE' + struct.pack('<BBHQQ', 0, level, len(children), _UNDEF, _UNDEF) + struct.pack('<Q', keys[0])
        for c, k in zip(children, keys[1:]):
            node += struct.pack('<QQ', c, k)
        node += b'\0' * (24 + 8 * (2 * self.INTERNAL_K + 1) + 8 * 2 * self.INTERNAL_K - len(node))
        return self.alloc(node)

    def finish(self, root):
        header, tree, heap = root
        sb = _H5_SIG + struct.pack('<BBBBBBBBHHI', 0, 0, 0, 0, 0, 8, 8, 0, self.LEAF_K, self.INTERNAL_K, 0)
        sb += struct.pack('<QQQQ', 0, _UNDEF, len(self.b), _UNDEF)
        sb += struct.pack('<QQII', 0, header, 1, 0) + struct.pack('<QQ', tree, heap)
        assert len(sb) == 96
        self.b[:96] = sb
        return bytes(self.b)


def write_hdf5(path, tree, chunks=None, attrs=None):
    """tree: nested dict {name: dict | ndarray} -> HDF5 file in the subset read_hdf5 understands.
    chunks {dataset name: chunk shape}: store those datasets chunked with shuffle + deflate instead of contiguous.
    attrs {group name: {attribute: str | bytes | float | int}}: attributes of the groups with that name (phrase dumps: context /
    title / offset / scale)."""
    w = _H5Writer()
    chunks = chunks or {}
    attrs = attrs or {}

    def emit(node, name=None):
        if isinstance(node, dict):
            return w.group({k: (emit(child, k)[0] if isinstance(child, dict) else emit(child, k)) for k, child in node.items()},
                           attrs.get(name))
        return w.dataset_chunked(node, chunks[name]) if name in chunks else w.dataset(node)

    data = w.finish(emit(tree))
    with open(path, 'wb') as f:
        f.write(data)
