"""Python face of the C++ host mirror (include/arroy_b200_host.h): the same objects and method
names a user of arroy works with — Writer / ArroyBuilder / Reader / QueryBuilder, StdRng — over an
in-memory Env that stores the reference's exact key/value bytes. All vector math runs on the GPU
through the C ABI; nothing here computes distances."""
import ctypes as C

import numpy as np

from . import _capi
from ._capi import METRICS, NODE_SINK, CANCEL_FN, _f32p, _u32p, _u64p, _u8p

KV_SINK = C.CFUNCTYPE(C.c_int32, C.c_void_p, _u8p, C.c_uint64, _u8p, C.c_uint64)
PROGRESS_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_char_p)

HOST_SIGNATURES = [
    ("arroy_host_last_error", C.c_char_p, []),
    ("arroy_env_new", C.c_void_p, []),
    ("arroy_env_free", None, [C.c_void_p]),
    ("arroy_env_len", C.c_uint64, [C.c_void_p]),
    ("arroy_env_iter", C.c_int32, [C.c_void_p, KV_SINK, C.c_void_p]),
    ("arroy_env_resident", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_env_put_raw", C.c_int32, [C.c_void_p, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64]),
    ("arroy_host_reencode", C.c_int32, [C.c_int32, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, _u64p]),
    ("arroy_rng_from_seed", C.c_void_p, [_u8p]),
    ("arroy_rng_seed_from_u64", C.c_void_p, [C.c_uint64]),
    ("arroy_rng_clone", C.c_void_p, [C.c_void_p]),
    ("arroy_rng_free", None, [C.c_void_p]),
    ("arroy_rng_next_u32", C.c_uint32, [C.c_void_p]),
    ("arroy_rng_gen_f32", C.c_float, [C.c_void_p]),
    ("arroy_rng_fill_f32", None, [C.c_void_p, _f32p, C.c_uint64]),
    ("arroy_writer_new", C.c_void_p, [C.c_void_p, C.c_uint16, C.c_uint32, C.c_int32]),
    ("arroy_writer_free", None, [C.c_void_p]),
    ("arroy_writer_add_item", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, C.c_uint32]),
    ("arroy_writer_add_items", C.c_int32, [C.c_void_p, C.c_uint64, _u32p, C.c_void_p]),
    ("arroy_writer_append_item", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, C.c_uint32]),
    ("arroy_writer_del_item", C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(C.c_int32)]),
    ("arroy_writer_clear", C.c_int32, [C.c_void_p]),
    ("arroy_writer_need_build", C.c_int32, [C.c_void_p, C.POINTER(C.c_int32)]),
    ("arroy_writer_contains_item", C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(C.c_int32)]),
    ("arroy_writer_is_empty", C.c_int32, [C.c_void_p, C.POINTER(C.c_int32)]),
    ("arroy_writer_item_vector", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, C.POINTER(C.c_int32)]),
    ("arroy_writer_build", C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_uint64, C.c_uint64, CANCEL_FN, C.c_void_p, PROGRESS_FN, C.c_void_p]),
    ("arroy_writer_build_timings", C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    ("arroy_reader_open", C.c_int32, [C.c_void_p, C.c_uint16, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    ("arroy_reader_free", None, [C.c_void_p]),
    ("arroy_reader_dimensions", C.c_uint32, [C.c_void_p]),
    ("arroy_reader_n_trees", C.c_uint64, [C.c_void_p]),
    ("arroy_reader_n_items", C.c_uint64, [C.c_void_p]),
    ("arroy_reader_item_ids", C.c_uint64, [C.c_void_p, _u32p, C.c_uint64]),
    ("arroy_reader_item_vector", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, C.POINTER(C.c_int32)]),
    ("arroy_reader_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_reader_nns_by_item", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, C.c_int64, _u32p, _f32p, _u64p, C.POINTER(C.c_int32)]),
    ("arroy_reader_nns_by_vector", C.c_int32, [C.c_void_p, _f32p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, C.c_int64, _u32p, _f32p, _u64p]),
    ("arroy_reader_nns_batch_by_item", C.c_int32, [C.c_void_p, C.c_uint32, _u32p, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, _f32p, _u32p, C.POINTER(C.c_double)]),
    ("arroy_reader_nns_batch", C.c_int32, [C.c_void_p, C.c_uint32, _u32p, _f32p, C.c_uint64, C.c_uint64, C.c_uint64, _u32p, C.c_int64, _u32p, _f32p, _u32p,
                                           C.POINTER(C.c_double)]),
    ("arroy_reader_nns_batch_multi", C.c_int32, [C.c_void_p, C.c_uint32, _u32p, _f32p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, _u64p, _u32p, _u32p,
                                                 _u32p, _f32p, _u32p, C.POINTER(C.c_double)]),
]

_BOUND = False


def _lib():
    global _BOUND
    lib = _capi.load()
    if not _BOUND:
        for name, res, args in HOST_SIGNATURES:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _BOUND = True
    return lib


def _id_array(ids):
    """A collection of item ids as a uint32 array (any order; the library sorts)."""
    a = ids if isinstance(ids, np.ndarray) else np.fromiter(ids, dtype=np.int64)
    a = a.ravel()
    if a.dtype != np.uint32:
        if a.size and (a.min() < 0 or a.max() > 0xffffffff):
            raise ValueError("item ids are u32")
        a = a.astype(np.uint32)
    return a


class ArroyError(RuntimeError):
    """arroy::Error (src/error.rs). `.kind` is the variant name."""
    KINDS = {100: "InvalidVecDimension", 101: "DatabaseFull", 102: "InvalidItemAppend", 103: "UnmatchingDistance", 104: "MissingMetadata",
             105: "NeedBuild", 106: "BuildCancelled", 107: "MissingKey", 108: "UnknownVersion", 109: "Panic",
             1: "Cuda", 2: "InvalidArgument", 3: "BuildCancelled", 4: "Capacity", 5: "NotStaged", 6: "Internal"}

    def __init__(self, code, message):
        super().__init__(message)
        self.code = code
        self.kind = self.KINDS.get(code, "Unknown")


def _ck(rc):
    if rc != 0:
        raise ArroyError(rc, _lib().arroy_host_last_error().decode())


class StdRng:
    """rand::rngs::StdRng (ChaCha12), product-side implementation."""

    def __init__(self, handle):
        self.h = handle

    @classmethod
    def from_seed(cls, seed):
        seed = bytes(seed)
        assert len(seed) == 32
        return cls(_lib().arroy_rng_from_seed((C.c_uint8 * 32)(*seed)))

    @classmethod
    def seed_from_u64(cls, state):
        return cls(_lib().arroy_rng_seed_from_u64(state))

    def clone(self):
        return StdRng(_lib().arroy_rng_clone(self.h))

    def __del__(self):
        try:
            _lib().arroy_rng_free(self.h)
        except Exception:
            pass

    def next_u32(self):
        return _lib().arroy_rng_next_u32(self.h)

    def gen_f32(self):
        return _lib().arroy_rng_gen_f32(self.h)

    def fill_f32(self, n):
        out = np.empty(n, dtype=np.float32)
        _lib().arroy_rng_fill_f32(self.h, out.ctypes.data_as(_f32p), n)
        return out


def reencode(what, value):
    """Decode `value` with the library's decoders and encode it again ('node' | 'metadata'): a faithful codec returns the input."""
    out = C.create_string_buffer(len(value) + 64)
    n = C.c_uint64(0)
    _ck(_lib().arroy_host_reencode(0 if what == "node" else 1, value, len(value), out, len(value) + 64, C.byref(n)))
    return out.raw[:n.value]


class Env:
    """Stands in for heed::Env + Database<D>: ordered key/value table + the GPU context."""

    def __init__(self, device=0):
        self.h = _lib().arroy_env_new()
        self.device = device
        self._ctx = None

    @property
    def ctx(self):
        if self._ctx is None:
            self._ctx = _capi.Context(self.device)  # raises without a CUDA device: no CPU fallback
        return self._ctx

    def __len__(self):
        return _lib().arroy_env_len(self.h)

    def items(self):
        """[(key bytes, value bytes)] in key order (what the reference's test dump iterates)."""
        out = []

        def sink(_a, k, kl, v, vl):
            out.append((C.string_at(k, kl), C.string_at(v, vl)))
            return 0

        cb = KV_SINK(sink)
        _ck(_lib().arroy_env_iter(self.h, cb, None))
        return out

    def put_raw(self, key, value):
        """Insert one (key, value) pair as is (importing the content of a real arroy LMDB file)."""
        _ck(_lib().arroy_env_put_raw(self.h, key, len(key), value, len(value)))

    def resident(self):
        """The table's record of the items it left on the device: None, or {"index", "epoch", "dirty"} (dirty = how many item
        ids were written or deleted since those rows were staged)."""
        out = (C.c_uint64 * 4)()
        _ck(_lib().arroy_env_resident(self.h, out))
        return {"index": int(out[1]), "epoch": int(out[2]), "dirty": int(out[3])} if out[0] else None

    def tree_nodes(self, index=0):
        """{node id: NodeCodec bytes} of one index."""
        out = {}
        for k, v in self.items():
            if int.from_bytes(k[0:2], "big") == index and k[2] == 2:
                out[int.from_bytes(k[3:7], "big")] = v
        return out

    def metadata(self, index=0):
        for k, v in self.items():
            if int.from_bytes(k[0:2], "big") == index and k[2] == 0 and int.from_bytes(k[3:7], "big") == 0:
                return v
        return None

    def close(self):
        if self._ctx is not None:
            self._ctx.close()
            self._ctx = None
        if self.h:
            _lib().arroy_env_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ArroyBuilder:
    """src/writer.rs:126-265"""

    def __init__(self, writer, rng):
        self.writer = writer
        self.rng = rng
        self._n_trees = None
        self._split_after = None
        self._available_memory = None
        self._cancel = None
        self._progress = None

    def n_trees(self, n):
        self._n_trees = n
        return self

    def split_after(self, n):
        self._split_after = n
        return self

    def available_memory(self, n):
        self._available_memory = n
        return self

    def cancel(self, fn):
        self._cancel = fn
        return self

    def progress(self, fn):
        self._progress = fn
        return self

    def build(self):
        w = self.writer
        ccb = CANCEL_FN((lambda _a: 1 if self._cancel() else 0)) if self._cancel else C.cast(None, CANCEL_FN)
        pcb = PROGRESS_FN((lambda _a, s: self._progress(s.decode()))) if self._progress else C.cast(None, PROGRESS_FN)
        # the build needs the device as soon as there is something to split or preprocess; tiny
        # indexes (one Descendants node) are pure host work, so a missing GPU only fails real builds
        try:
            ctx_h = w.env.ctx.h
        except _capi.ArroyB200Error:
            ctx_h = None
        _ck(_lib().arroy_writer_build(w.h, ctx_h, self.rng.h, -1 if self._n_trees is None else self._n_trees, self._split_after or 0,
                                      (2**64 - 1) if self._available_memory is None else self._available_memory, ccb, None, pcb, None))


class Writer:
    """src/writer.rs:268-485"""

    def __init__(self, env, index, dimensions, distance):
        self.env = env
        self.index = index
        self.dimensions = dimensions
        self.metric = METRICS[distance] if isinstance(distance, str) else distance
        self.h = _lib().arroy_writer_new(env.h, index, dimensions, self.metric)

    def __del__(self):
        try:
            _lib().arroy_writer_free(self.h)
        except Exception:
            pass

    def add_item(self, item, vector):
        v = np.ascontiguousarray(vector, dtype=np.float32)
        _ck(_lib().arroy_writer_add_item(self.h, item, v.ctypes.data_as(_f32p), v.size))

    def add_items(self, items, vectors):
        items = np.ascontiguousarray(items, dtype=np.uint32)
        if hasattr(vectors, "data_ptr"):
            assert vectors.shape[1] == self.dimensions
            ptr = vectors.data_ptr()
        else:
            vectors = np.ascontiguousarray(vectors, dtype=np.float32)
            assert vectors.shape[1] == self.dimensions
            ptr = vectors.ctypes.data
        _ck(_lib().arroy_writer_add_items(self.h, items.size, items.ctypes.data_as(_u32p), C.c_void_p(ptr)))

    def append_item(self, item, vector):
        v = np.ascontiguousarray(vector, dtype=np.float32)
        _ck(_lib().arroy_writer_append_item(self.h, item, v.ctypes.data_as(_f32p), v.size))

    def del_item(self, item):
        ex = C.c_int32(0)
        _ck(_lib().arroy_writer_del_item(self.h, item, C.byref(ex)))
        return bool(ex.value)

    def clear(self):
        _ck(_lib().arroy_writer_clear(self.h))

    def need_build(self):
        o = C.c_int32(0)
        _ck(_lib().arroy_writer_need_build(self.h, C.byref(o)))
        return bool(o.value)

    def contains_item(self, item):
        o = C.c_int32(0)
        _ck(_lib().arroy_writer_contains_item(self.h, item, C.byref(o)))
        return bool(o.value)

    def is_empty(self):
        o = C.c_int32(0)
        _ck(_lib().arroy_writer_is_empty(self.h, C.byref(o)))
        return bool(o.value)

    def item_vector(self, item):
        out = np.empty(self.dimensions, dtype=np.float32)
        f = C.c_int32(0)
        _ck(_lib().arroy_writer_item_vector(self.h, item, out.ctypes.data_as(_f32p), C.byref(f)))
        return out if f.value else None

    def builder(self, rng):
        return ArroyBuilder(self, rng)

    def build_timings(self):
        t = (C.c_double * 8)()
        _lib().arroy_writer_build_timings(self.h, t)
        keys = ["stage_ms", "preprocess_ms", "build_ms", "metadata_ms", "total_ms", "h2d_bytes", "node_bytes", "reserved"]
        return dict(zip(keys, list(t)))


class QueryBuilder:
    """src/reader.rs:26-124"""

    def __init__(self, reader, count):
        self.reader = reader
        self.count = count
        self._search_k = None
        self._oversampling = None
        self._candidates = None

    def search_k(self, n):
        self._search_k = n
        return self

    def oversampling(self, n):
        self._oversampling = n
        return self

    def candidates(self, ids):
        self._candidates = np.ascontiguousarray(sorted(ids), dtype=np.uint32)
        return self

    def _cand(self):
        if self._candidates is None:
            return None, -1
        return self._candidates.ctypes.data_as(_u32p), self._candidates.size

    def by_item(self, item):
        out_ids = np.empty(max(self.count, 1), dtype=np.uint32)
        out_dist = np.empty(max(self.count, 1), dtype=np.float32)
        n = C.c_uint64(0)
        found = C.c_int32(0)
        cp, cn = self._cand()
        _ck(_lib().arroy_reader_nns_by_item(self.reader.h, item, self.count, min(self._search_k or 0, 2**64 - 1), self._oversampling or 0, cp, cn,
                                            out_ids.ctypes.data_as(_u32p), out_dist.ctypes.data_as(_f32p), C.byref(n), C.byref(found)))
        if not found.value:
            return None
        return list(zip(out_ids[:n.value].tolist(), out_dist[:n.value].tolist()))

    def by_vector(self, vector):
        v = np.ascontiguousarray(vector, dtype=np.float32)
        out_ids = np.empty(max(self.count, 1), dtype=np.uint32)
        out_dist = np.empty(max(self.count, 1), dtype=np.float32)
        n = C.c_uint64(0)
        cp, cn = self._cand()
        _ck(_lib().arroy_reader_nns_by_vector(self.reader.h, v.ctypes.data_as(_f32p), v.size, self.count, min(self._search_k or 0, 2**64 - 1),
                                              self._oversampling or 0, cp, cn, out_ids.ctypes.data_as(_u32p), out_dist.ctypes.data_as(_f32p), C.byref(n)))
        return list(zip(out_ids[:n.value].tolist(), out_dist[:n.value].tolist()))


class Reader:
    """src/reader.rs:138-298"""

    def __init__(self, handle, env, index=0):
        self.h = handle
        self.env = env
        self._index = index

    @classmethod
    def open(cls, env, index, distance):
        metric = METRICS[distance] if isinstance(distance, str) else distance
        h = C.c_void_p()
        # the context handle is needed only once a query has candidates to re-rank; creating it
        # lazily keeps error paths (MissingMetadata, NeedBuild, ...) testable without a GPU
        ctx_h = env._ctx.h if env._ctx is not None else None
        if ctx_h is None:
            try:
                ctx_h = env.ctx.h
            except _capi.ArroyB200Error:
                ctx_h = None
        _ck(_lib().arroy_reader_open(env.h, index, metric, ctx_h, C.byref(h)))
        return cls(h, env, index)

    def __del__(self):
        try:
            _lib().arroy_reader_free(self.h)
        except Exception:
            pass

    def dimensions(self):
        return _lib().arroy_reader_dimensions(self.h)

    def n_trees(self):
        return _lib().arroy_reader_n_trees(self.h)

    def n_items(self):
        return _lib().arroy_reader_n_items(self.h)

    def item_ids(self):
        n = _lib().arroy_reader_item_ids(self.h, None, 0)
        out = np.empty(n, dtype=np.uint32)
        _lib().arroy_reader_item_ids(self.h, out.ctypes.data_as(_u32p), n)
        return out.tolist()

    def item_vector(self, item):
        out = np.empty(self.dimensions(), dtype=np.float32)
        f = C.c_int32(0)
        _ck(_lib().arroy_reader_item_vector(self.h, item, out.ctypes.data_as(_f32p), C.byref(f)))
        return out if f.value else None

    def _roots(self):
        m = self.env.metadata(self._index)
        z = m.index(b"\x00")
        size = int.from_bytes(m[z + 5:z + 9], "big")
        return np.frombuffer(m[z + 9 + size:], dtype=np.uint32).tolist()

    def stats(self):
        t = self.n_trees()
        out = np.zeros(4 * max(t, 1), dtype=np.uint64)
        _ck(_lib().arroy_reader_stats(self.h, out.ctypes.data_as(_u64p)))
        keys = ("depth", "dummy_normals", "split_nodes", "descendants")
        return {"leaf": self.n_items(), "tree_stats": [dict(zip(keys, out[4 * i:4 * i + 4].tolist())) for i in range(t)]}

    def nns(self, count):
        return QueryBuilder(self, count)

    def nns_batch_by_item(self, items, count, search_k=None, oversampling=None, candidates=None, filters=None, filter_of_query=None):
        """One nns(count).search_k(..).oversampling(..).candidates(..).by_item(it) per item, in one call; candidates (optional)
        is shared by every query. Or one filter per query: filters is a list of id collections and query i uses
        filters[filter_of_query[i]] (not together with candidates). Returns (ids nq x count, distances nq x count, lengths nq,
        timings)."""
        items = np.ascontiguousarray(items, dtype=np.uint32)
        return self._nns_batch(items.size, items.ctypes.data_as(_u32p), None, count, search_k, oversampling, candidates, filters, filter_of_query, items)

    def nns_batch_by_vector(self, vectors, count, search_k=None, oversampling=None, candidates=None, filters=None, filter_of_query=None):
        """nns_batch_by_item for query vectors (nq x dimensions), as QueryBuilder::by_vector."""
        vectors = np.ascontiguousarray(vectors, dtype=np.float32)
        if vectors.ndim != 2 or vectors.shape[1] != self.dimensions():
            raise ArroyError(100, "Invalid vector dimensions. Got %s but expected %d" % (vectors.shape[1:] or vectors.shape, self.dimensions()))
        return self._nns_batch(vectors.shape[0], None, vectors.ctypes.data_as(_f32p), count, search_k, oversampling, candidates, filters, filter_of_query,
                               vectors)

    def _nns_batch(self, nq, items_p, vectors_p, count, search_k, oversampling, candidates, filters, filter_of_query, _keep):
        out_ids = np.zeros((nq, max(count, 1)), dtype=np.uint32)
        out_dist = np.zeros((nq, max(count, 1)), dtype=np.float32)
        out_len = np.zeros(nq, dtype=np.uint32)
        ms = (C.c_double * 2)()
        sk, os_ = min(search_k or 0, 2**64 - 1), oversampling or 0
        outs = (out_ids.ctypes.data_as(_u32p), out_dist.ctypes.data_as(_f32p), out_len.ctypes.data_as(_u32p), ms)
        if filters is not None or filter_of_query is not None:
            if candidates is not None:
                raise ValueError("candidates= is one filter for every query; filters= / filter_of_query= give each query its own: pass one or the other")
            if filters is None or filter_of_query is None:
                raise ValueError("filters= and filter_of_query= go together")
            lists = [_id_array(f) for f in filters]
            offsets = np.zeros(len(lists) + 1, dtype=np.uint64)
            offsets[1:] = np.cumsum([f.size for f in lists])
            ids = np.concatenate(lists) if lists else np.zeros(0, np.uint32)
            fq = np.ascontiguousarray(filter_of_query, dtype=np.uint32)
            if fq.size != nq:
                raise ValueError("filter_of_query must hold one filter index per query (%d)" % nq)
            _ck(_lib().arroy_reader_nns_batch_multi(self.h, nq, items_p, vectors_p, count, sk, os_, len(lists), offsets.ctypes.data_as(_u64p),
                                                    ids.ctypes.data_as(_u32p), fq.ctypes.data_as(_u32p), *outs))
        else:
            cand = None if candidates is None else np.ascontiguousarray(sorted(candidates), dtype=np.uint32)
            _ck(_lib().arroy_reader_nns_batch(self.h, nq, items_p, vectors_p, count, sk, os_, None if cand is None else cand.ctypes.data_as(_u32p),
                                              -1 if cand is None else cand.size, *outs))
        return out_ids, out_dist, out_len, {"tree_walk_ms": ms[0], "rerank_ms": ms[1]}
