"""ctypes binding of include/arroy_b200.h (libarroy_b200.so, built in-tree by
__graft_entry__.build()). No fallback: if the library or a CUDA device is missing, calls
raise — nothing here computes on the CPU."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ARROY_B200_LIB") or os.path.join(_HERE, "libarroy_b200.so")   # (override: A/B runs of two builds)

EUCLIDEAN, COSINE, DOT_PRODUCT, MANHATTAN = 0, 1, 2, 3
BQ_EUCLIDEAN, BQ_COSINE, BQ_MANHATTAN = 4, 5, 6
METRICS = {"euclidean": 0, "cosine": 1, "dot-product": 2, "manhattan": 3,
           "binary quantized euclidean": 4, "binary quantized cosine": 5, "binary quantized manhattan": 6}
METRIC_NAMES = {v: k for k, v in METRICS.items()}

OK, ERR_CUDA, ERR_INVALID, ERR_CANCELLED, ERR_CAPACITY, ERR_NOT_STAGED, ERR_INTERNAL = range(7)

_f32p = C.POINTER(C.c_float)
_u32p = C.POINTER(C.c_uint32)
_u64p = C.POINTER(C.c_uint64)
_u8p = C.POINTER(C.c_uint8)
NODE_SINK = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_uint32, _u8p, C.c_uint64)
CANCEL_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p)

# every symbol include/arroy_b200.h declares: (name, restype, argtypes)
SIGNATURES = [
    ("arroy_b200_version", C.c_char_p, []),
    ("arroy_b200_allocations", C.c_int32, [_u64p]),
    ("arroy_b200_create", C.c_int32, [C.c_int32, C.POINTER(C.c_void_p)]),
    ("arroy_b200_destroy", None, [C.c_void_p]),
    ("arroy_b200_last_error", C.c_char_p, [C.c_void_p]),
    ("arroy_b200_stage_items", C.c_int32, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, _u32p, C.POINTER(C.c_void_p)]),
    ("arroy_b200_stage_items_delta", C.c_int32, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, _u32p, C.POINTER(C.c_void_p), C.c_uint64, _u32p]),
    ("arroy_b200_stage_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_read_items", C.c_int32, [C.c_void_p, _u32p, C.c_uint64, C.c_void_p]),
    ("arroy_b200_stage_delta_plan", C.c_uint64, [_u32p, C.c_uint64, _u32p, C.c_uint64, _u32p, C.c_uint64, C.POINTER(C.c_int64)]),
    ("arroy_b200_item_placement_plan", C.c_uint32, [C.c_int32, C.c_uint32, C.c_uint64, C.c_uint64]),
    ("arroy_b200_item_placement", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_stage_items_flat", C.c_int32, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, _u32p, C.c_void_p, _f32p, _f32p]),
    ("arroy_b200_stage_items_device", C.c_int32, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, _u32p, C.c_void_p]),
    ("arroy_b200_item_headers", C.c_int32, [C.c_void_p, _f32p, _f32p]),
    ("arroy_b200_dot_preprocess", C.c_int32, [C.c_void_p, _f32p, _f32p]),
    ("arroy_b200_side_batch", C.c_int32, [C.c_void_p, _f32p, C.c_float, C.c_float, _u32p, C.c_uint64, _u8p, _f32p]),
    ("arroy_b200_side_multi", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, _f32p, _f32p, _u32p, _u64p, _u8p]),
    ("arroy_b200_create_split", C.c_int32, [C.c_void_p, _u32p, _u64p, _u32p, C.c_uint64, _f32p, _f32p]),
    ("arroy_b200_build_trees", C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, _u32p, C.c_uint32, C.c_uint32, CANCEL_FN, C.c_void_p, NODE_SINK, C.c_void_p, _u64p]),
    ("arroy_b200_build_trees_begin", C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, CANCEL_FN, C.c_void_p, _u32p]),
    ("arroy_b200_build_trees_emit", C.c_int32, [C.c_void_p, _u32p, _u64p, NODE_SINK, C.c_void_p]),
    ("arroy_b200_build_subtrees_begin", C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, _u32p, _u64p, C.c_uint32, CANCEL_FN, C.c_void_p, _u32p]),
    ("arroy_b200_build_subtrees_begin_at", C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, _u64p, _u32p, _u64p, C.c_uint32, CANCEL_FN, C.c_void_p, _u32p, _u64p]),
    ("arroy_b200_build_trees_emit_mapped", C.c_int32, [C.c_void_p, _u32p, _u32p, NODE_SINK, C.c_void_p]),
    ("arroy_b200_build_stats", C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    ("arroy_b200_rerank", C.c_int32, [C.c_void_p, _f32p, C.c_float, C.c_float, _u32p, C.c_uint64, C.c_uint32, _u32p, _f32p, _u32p]),
    ("arroy_b200_rerank_batch", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, _f32p, _f32p, _u32p, _u64p, C.c_uint32, _u32p, _f32p, _u32p]),
    ("arroy_b200_rerank_shared", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, _f32p, _u32p, C.c_uint64, C.c_uint32, _u32p, _f32p, _u32p]),
    ("arroy_b200_load_forest", C.c_int32, [C.c_void_p, C.c_uint32, _u8p, _u32p, _u32p, _u32p, _f32p, _u32p, _u32p, C.c_uint32, _f32p, C.c_uint64, _u32p, C.c_uint32, _u32p]),
    ("arroy_b200_search_batch", C.c_int32, [C.c_void_p, C.c_uint32, _u32p, _f32p, _f32p, C.c_uint64, C.c_uint64, _u32p, _f32p, _u32p, C.POINTER(C.c_int32)]),
    ("arroy_b200_search_batch_filtered", C.c_int32, [C.c_void_p, C.c_uint32, _u32p, _f32p, _f32p, C.c_uint64, C.c_uint64, _u32p, _u32p, _f32p, _u32p, C.POINTER(C.c_int32)]),
    ("arroy_b200_search_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_search_batch_multi_filtered", C.c_int32, [C.c_void_p, C.c_uint32, _u32p, _f32p, _f32p, C.c_uint64, C.c_uint64, C.c_uint32, _u64p, _u32p, _u32p,
                                                           _u32p, _f32p, _u32p, C.POINTER(C.c_int32)]),
    ("arroy_b200_multi_filter_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_synth_device", C.c_int32, [C.c_void_p, _u8p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_float, C.c_void_p]),
    ("arroy_b200_time_scan", C.c_int32, [C.c_void_p, _f32p, C.c_float, C.c_float, _u32p, C.c_uint64, C.c_int32, C.c_int32, C.c_int32, _f32p, _u64p]),
    ("arroy_b200_arena_new", C.c_void_p, []),
    ("arroy_b200_arena_free", None, [C.c_void_p]),
    ("arroy_b200_arena_clear", None, [C.c_void_p]),
    ("arroy_b200_arena_sink", C.c_int32, [C.c_void_p, C.c_uint32, _u8p, C.c_uint64]),
    ("arroy_b200_arena_stats", C.c_uint64, [C.c_void_p, _u64p]),
    ("arroy_b200_arena_get", C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(_u8p), _u64p]),
    ("arroy_b200_build_breakdown", C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    ("arroy_b200_counters", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_plane_rerank_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_rerank_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_rerank_breakdown", C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    ("arroy_b200_search_breakdown", C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    ("arroy_b200_prefilter_scores", C.c_int32, [C.c_void_p, C.c_uint32, _f32p, _u32p, C.c_uint64, C.c_int32, _f32p]),
    ("arroy_b200_timer_start", C.c_int32, [C.c_void_p]),
    ("arroy_b200_timer_stop", C.c_int32, [C.c_void_p, _f32p]),
    ("arroy_b200_device_ptrs", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), _u32p]),
    ("arroy_b200_epochs", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_bq_quantize", C.c_uint32, [_f32p, C.c_uint32, _f32p]),
    ("arroy_b200_build_shadow_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_build_prefilter_stats", C.c_int32, [C.c_void_p, _u64p]),
    ("arroy_b200_prefilter_planes", C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, _f32p]),
    ("arroy_b200_selftest_udiv", C.c_int32, [C.c_void_p, C.c_uint64, C.c_uint64, _u64p, _u64p]),
    ("arroy_b200_stage_begin", C.c_int32, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, _u32p]),
    ("arroy_b200_stage_rows", C.c_int32, [C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_void_p)]),
    ("arroy_b200_stage_end", C.c_int32, [C.c_void_p, C.c_int32]),
    ("arroy_b200_create_group", C.c_int32, [C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]),
    ("arroy_b200_destroy_group", None, [C.c_void_p]),
    ("arroy_b200_group_last_error", C.c_char_p, [C.c_void_p]),
    ("arroy_b200_group_size", C.c_int32, [C.c_void_p]),
    ("arroy_b200_group_ctx", C.c_void_p, [C.c_void_p, C.c_int32]),
    ("arroy_b200_group_stage_items", C.c_int32, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, _u32p, C.POINTER(C.c_void_p)]),
    ("arroy_b200_group_dot_preprocess", C.c_int32, [C.c_void_p, _f32p, _f32p]),
    ("arroy_b200_group_build_trees", C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, _u32p, C.c_uint32, C.c_uint32, CANCEL_FN, C.c_void_p, NODE_SINK, C.c_void_p, _u64p]),
    ("arroy_b200_group_stage_breakdown", C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
]

_LIB = None


class ArroyB200Error(RuntimeError):
    def __init__(self, code, message):
        super().__init__("arroy_b200 error %d: %s" % (code, message))
        self.code = code
        self.message = message


def load():
    """Load the shared library (no CUDA call is made by loading)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("%s is missing — run `python -c 'import __graft_entry__ as g; g.build()'`" % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, res, args in SIGNATURES:
            if os.environ.get("ARROY_B200_LIB") and not hasattr(lib, name):
                continue   # an older build loaded for an A/B run
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


def _fp(a):
    return a.ctypes.data_as(_f32p) if a is not None else None


def _up(a):
    return a.ctypes.data_as(_u32p) if a is not None else None


def row_bitmap(rows, n):
    """The filter arroy_b200_search_batch_filtered takes: ceil(n / 32) uint32 words, bit r set for every r in rows (< n)."""
    bits = np.zeros(((n + 31) // 32) * 32, dtype=bool)
    bits[np.asarray(rows, dtype=np.int64)] = True
    return np.packbits(bits, bitorder="little").view("<u4").astype(np.uint32)


def bq_quantize(vector):
    """BinaryQuantized::from_slice + ::iter of one vector: its +-1.0 values, padded to a multiple of 64 (host helper)."""
    v = np.ascontiguousarray(vector, dtype=np.float32)
    out = np.empty((v.size + 63) // 64 * 64, dtype=np.float32)
    load().arroy_b200_bq_quantize(_fp(v), v.size, _fp(out))
    return out


def stage_delta_plan(old_ids, new_ids, changed_ids):
    """The plan of Context.stage_items_delta (host only): for every row of new_ids the row of old_ids it keeps, -1 = uploaded.
    Returns (src int64 array, number of uploaded rows). The three id lists ascend strictly."""
    old, new, ch = (np.ascontiguousarray(a, dtype=np.uint32) for a in (old_ids, new_ids, changed_ids))
    src = np.empty(new.size, dtype=np.int64)
    n = load().arroy_b200_stage_delta_plan(_up(old), old.size, _up(new), new.size, _up(ch), ch.size, src.ctypes.data_as(C.POINTER(C.c_int64)))
    return src, int(n)


def allocations():
    """What the library holds now, in the whole process (arroy_b200_allocations; no CUDA call)."""
    out = (C.c_uint64 * 5)()
    load().arroy_b200_allocations(out)
    return dict(zip(["device_buffers", "device_bytes", "pinned_buffers", "pinned_bytes", "handles"], (int(v) for v in out)))


def item_placement_plan(metric, dim, n, free_bytes):
    """Where stage_items_ptrs / stage_items_flat put an index's f32 rows given free_bytes of device memory (host only):
    "device", or "host" (mapped pinned host memory; the device keeps the 8-bit planes)."""
    metric = METRICS[metric] if isinstance(metric, str) else metric
    return "host" if load().arroy_b200_item_placement_plan(metric, dim, n, free_bytes) == 1 else "device"


class Context:
    """One arroy_ctx (one GPU). Thin 1:1 wrapper over the C ABI."""

    def __init__(self, device=0):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.arroy_b200_create(device, C.byref(h))
        if rc != OK:
            raise ArroyB200Error(rc, "arroy_b200_create failed (no CUDA device / library not built for this GPU)")
        self.h = h
        self.device = device
        self.n = 0
        self.dim = 0
        self.metric = None

    def close(self):
        if getattr(self, "h", None):
            self.lib.arroy_b200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != OK:
            raise ArroyB200Error(rc, self.lib.arroy_b200_last_error(self.h).decode())

    def _staged(self, n, dim, metric):
        # binary-quantized metrics: vectors cross the boundary as their +-1 values, padded to a multiple of 64
        self.n, self.metric, self.user_dim = n, metric, dim
        self.dim = (dim + 63) // 64 * 64 if metric is not None and metric >= BQ_EUCLIDEAN else dim

    # -- staging ---------------------------------------------------------------------------
    def stage_items_flat(self, metric, ids, vectors, hdr0=None, hdr1=None):
        metric = METRICS[metric] if isinstance(metric, str) else metric
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        if hasattr(vectors, "data_ptr"):  # torch CPU tensor (possibly pinned)
            n, dim = vectors.shape
            ptr = vectors.data_ptr()
            keep = vectors
        else:
            vectors = np.ascontiguousarray(vectors, dtype=np.float32)
            n, dim = vectors.shape
            ptr = vectors.ctypes.data
            keep = vectors
        assert ids.size == n
        h0 = None if hdr0 is None else np.ascontiguousarray(hdr0, dtype=np.float32)
        h1 = None if hdr1 is None else np.ascontiguousarray(hdr1, dtype=np.float32)
        self._ck(self.lib.arroy_b200_stage_items_flat(self.h, metric, dim, n, _up(ids), C.c_void_p(ptr), _fp(h0), _fp(h1)))
        del keep
        self._staged(n, dim, metric)

    def stage_items_leaf_values(self, metric, dim, ids, values):
        """values: list of bytes objects = raw stored Leaf values ([0x00][header][dim x f32])."""
        metric = METRICS[metric] if isinstance(metric, str) else metric
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        n = ids.size
        bufs = [C.create_string_buffer(v, len(v)) for v in values]
        arr = (C.c_void_p * max(n, 1))(*[C.cast(b, C.c_void_p) for b in bufs])
        self._ck(self.lib.arroy_b200_stage_items(self.h, metric, dim, n, _up(ids), arr))
        self._staged(n, dim, metric)

    def stage_items_device(self, metric, ids, dim, device_ptr):
        metric = METRICS[metric] if isinstance(metric, str) else metric
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        self._ck(self.lib.arroy_b200_stage_items_device(self.h, metric, dim, ids.size, _up(ids), C.c_void_p(device_ptr)))
        self._staged(ids.size, dim, metric)

    def item_headers(self):
        h0 = np.empty(self.n, dtype=np.float32)
        h1 = np.empty(self.n, dtype=np.float32)
        self._ck(self.lib.arroy_b200_item_headers(self.h, _fp(h0), _fp(h1)))
        return h0, h1

    def dot_preprocess(self):
        extra = np.empty(self.n, dtype=np.float32)
        norm = np.empty(self.n, dtype=np.float32)
        self._ck(self.lib.arroy_b200_dot_preprocess(self.h, _fp(extra), _fp(norm)))
        return extra, norm

    # -- side / split ------------------------------------------------------------------------
    def side_batch(self, normal, hdr, rows, want_margin=True):
        normal = np.ascontiguousarray(normal, dtype=np.float32)
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        side = np.empty(rows.size, dtype=np.uint8)
        mg = np.empty(rows.size, dtype=np.float32) if want_margin else None
        self._ck(self.lib.arroy_b200_side_batch(self.h, _fp(normal), hdr[0], hdr[1], _up(rows), rows.size,
                                                side.ctypes.data_as(_u8p), _fp(mg)))
        return side, mg

    def create_split(self, key_words, word_pos, rows):
        key = np.ascontiguousarray(key_words, dtype=np.uint32)
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        pos = C.c_uint64(word_pos)
        normal = np.empty(self.dim, dtype=np.float32)
        hdr = np.zeros(2, dtype=np.float32)
        self._ck(self.lib.arroy_b200_create_split(self.h, _up(key), C.byref(pos), _up(rows), rows.size, _fp(normal), _fp(hdr)))
        return normal, (float(hdr[0]), float(hdr[1])), pos.value

    # -- forest --------------------------------------------------------------------------------
    def build_trees(self, tree_seeds, root_ids, first_free_node_id, split_after=0, cancel=None, collect=True):
        """Returns {node_id: NodeCodec bytes} (or the node count when collect=False)."""
        n_trees = len(tree_seeds)
        seeds = (C.c_uint8 * (32 * max(n_trees, 1)))()
        for t, s in enumerate(tree_seeds):
            assert len(s) == 32
            seeds[32 * t:32 * t + 32] = list(s)
        roots = np.ascontiguousarray(root_ids, dtype=np.uint32)
        out = {}

        def sink(_arg, node_id, ptr, length):
            out[node_id] = C.string_at(ptr, length)
            return 0

        cb = NODE_SINK(sink) if collect else C.cast(None, NODE_SINK)
        ccb = CANCEL_FN((lambda _a: 1 if cancel() else 0)) if cancel else C.cast(None, CANCEL_FN)
        n_nodes = C.c_uint64(0)
        self._ck(self.lib.arroy_b200_build_trees(self.h, n_trees, C.cast(seeds, C.c_void_p), _up(roots), first_free_node_id, split_after,
                                                 ccb, None, cb, None, C.byref(n_nodes)))
        return out if collect else n_nodes.value

    def build_trees_begin(self, tree_seeds, split_after=0):
        """Phase 1 of a sharded build: device work for the given (local) trees; returns node counts."""
        n_trees = len(tree_seeds)
        seeds = (C.c_uint8 * (32 * max(n_trees, 1)))()
        for t, s in enumerate(tree_seeds):
            seeds[32 * t:32 * t + 32] = list(s)
        counts = np.zeros(max(n_trees, 1), dtype=np.uint32)
        self._ck(self.lib.arroy_b200_build_trees_begin(self.h, n_trees, C.cast(seeds, C.c_void_p), split_after, C.cast(None, CANCEL_FN), None, _up(counts)))
        return counts[:n_trees]

    def build_trees_emit(self, root_ids, base_ids, arena=None):
        """Phase 2: encode the parked trees. Returns {node id: bytes} unless an Arena is given."""
        roots = np.ascontiguousarray(root_ids, dtype=np.uint32)
        bases = np.ascontiguousarray(base_ids, dtype=np.uint64)
        if arena is not None:
            sink = C.cast(self.lib.arroy_b200_arena_sink, NODE_SINK)
            self._ck(self.lib.arroy_b200_build_trees_emit(self.h, _up(roots), bases.ctypes.data_as(_u64p), sink, arena.h))
            return None
        out = {}

        def sink(_arg, node_id, ptr, length):
            out[node_id] = C.string_at(ptr, length)
            return 0

        cb = NODE_SINK(sink)
        self._ck(self.lib.arroy_b200_build_trees_emit(self.h, _up(roots), bases.ctypes.data_as(_u64p), cb, None))
        return out

    def build_trees_into_arena(self, arena, tree_seeds, root_ids, first_free_node_id, split_after=0):
        """C-level path: the library's own thread-safe arena sink (no Python callback)."""
        n_trees = len(tree_seeds)
        seeds = (C.c_uint8 * (32 * max(n_trees, 1)))()
        for t, s in enumerate(tree_seeds):
            seeds[32 * t:32 * t + 32] = list(s)
        roots = np.ascontiguousarray(root_ids, dtype=np.uint32)
        n_nodes = C.c_uint64(0)
        sink = C.cast(self.lib.arroy_b200_arena_sink, NODE_SINK)
        self._ck(self.lib.arroy_b200_build_trees(self.h, n_trees, C.cast(seeds, C.c_void_p), _up(roots), first_free_node_id, split_after,
                                                 C.cast(None, CANCEL_FN), None, sink, arena.h, C.byref(n_nodes)))
        return n_nodes.value

    def stage_items_ptrs(self, metric, dim, ids, ptr_array):
        """ptr_array: numpy uint64 array of host addresses of raw Leaf values (LMDB-style)."""
        metric = METRICS[metric] if isinstance(metric, str) else metric
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        ptrs = np.ascontiguousarray(ptr_array, dtype=np.uint64)
        self._ck(self.lib.arroy_b200_stage_items(self.h, metric, dim, ids.size, _up(ids), ptrs.ctypes.data_as(C.POINTER(C.c_void_p))))
        self._staged(ids.size, dim, metric)

    def stage_items_delta(self, metric, dim, ids, ptr_array, changed_ids):
        """stage_items_ptrs that keeps the resident rows of every id not in changed_ids (ascending); see stage_stats()."""
        metric = METRICS[metric] if isinstance(metric, str) else metric
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        ptrs = np.ascontiguousarray(ptr_array, dtype=np.uint64)
        ch = np.ascontiguousarray(changed_ids, dtype=np.uint32)
        self._ck(self.lib.arroy_b200_stage_items_delta(self.h, metric, dim, ids.size, _up(ids), ptrs.ctypes.data_as(C.POINTER(C.c_void_p)), ch.size, _up(ch)))
        self._staged(ids.size, dim, metric)

    def stage_stats(self):
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.arroy_b200_stage_stats(self.h, out))
        return {"uploaded_rows": int(out[0]), "moved_rows": int(out[1]), "delta": int(out[2]), "h2d_bytes": int(out[3])}

    def item_placement(self):
        """Where the staged f32 rows live: {"placement": "device" | "host", "device_bytes": device bytes held for item data (the
        rows, or the 8-bit planes and scales of host-placed rows), "host_bytes": pinned host bytes of the rows}."""
        out = (C.c_uint64 * 3)()
        self._ck(self.lib.arroy_b200_item_placement(self.h, out))
        return {"placement": "host" if out[0] == 1 else "device", "device_bytes": int(out[1]), "host_bytes": int(out[2])}

    def read_items(self, rows=None):
        """The raw resident rows (all of them by default) as a uint8 array n_rows x row_bytes, padding included."""
        rows = np.arange(self.n, dtype=np.uint32) if rows is None else np.ascontiguousarray(rows, dtype=np.uint32)
        if self.metric is not None and self.metric >= BQ_EUCLIDEAN:
            row_bytes = 16 * ((self.dim + 127) // 128)   # the bit string (arroy_b200_device_ptrs)
        else:
            row_bytes = 4 * ((self.dim + 31) // 32 * 32)
        out = np.empty((rows.size, row_bytes), dtype=np.uint8)
        self._ck(self.lib.arroy_b200_read_items(self.h, _up(rows), rows.size, out.ctypes.data))
        return out

    def stage_begin(self, metric, dim, ids):
        metric = METRICS[metric] if isinstance(metric, str) else metric
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        self._ck(self.lib.arroy_b200_stage_begin(self.h, metric, dim, ids.size, _up(ids)))
        self._staged(ids.size, dim, metric)

    def stage_rows(self, row0, ptr_array):
        ptrs = np.ascontiguousarray(ptr_array, dtype=np.uint64)
        self._ck(self.lib.arroy_b200_stage_rows(self.h, row0, ptrs.size, ptrs.ctypes.data_as(C.POINTER(C.c_void_p))))

    def stage_end(self, headers_on_device=False):
        self._ck(self.lib.arroy_b200_stage_end(self.h, 1 if headers_on_device else 0))

    def build_shadow_stats(self):
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.arroy_b200_build_shadow_stats(self.h, out))
        return {"rows_via_bf16_shadow": int(out[0]), "rows_rescored_f32": int(out[1]), "rows_in_fused_root_pass": int(out[2]), "fused_root_rows_read": int(out[3])}

    def build_prefilter_stats(self):
        """Rows of the last build through each stage of side()'s 8-bit pre-filter: all of them read the hi plane (d bytes), the
        stage-1 leftovers read the lo plane, the stage-2 leftovers the f32 row."""
        out = (C.c_uint64 * 5)()
        self._ck(self.lib.arroy_b200_build_prefilter_stats(self.h, out))
        return {"rows_via_prefilter": int(out[0]), "rows_stage2": int(out[1]), "rows_rescored_f32": int(out[2]),
                "rows_in_fused_root_pass": int(out[3]), "fused_root_rows_read": int(out[4])}

    def prefilter_planes(self, n, ld):
        """The pre-filter's encoding of the staged items: (hi int8 n x ld, lo int8 n x ld, scale f32 n)."""
        hi = np.empty((n, ld), dtype=np.int8)
        lo = np.empty((n, ld), dtype=np.int8)
        scale = np.empty(n, dtype=np.float32)
        self._ck(self.lib.arroy_b200_prefilter_planes(self.h, hi.ctypes.data, lo.ctypes.data, scale.ctypes.data_as(_f32p)))
        return hi, lo, scale

    def build_stats(self):
        st = (C.c_double * 8)()
        self._ck(self.lib.arroy_b200_build_stats(self.h, st))
        keys = ["scanned_rows", "steps", "create_split_calls", "random_splits", "build_ms", "scan_ms", "nodes", "misspeculated_splits"]
        return dict(zip(keys, list(st)))

    # -- re-rank -------------------------------------------------------------------------------
    def rerank(self, query, qhdr, rows, k):
        query = np.ascontiguousarray(query, dtype=np.float32)
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        out_rows = np.empty(max(k, 1), dtype=np.uint32)
        out_dist = np.empty(max(k, 1), dtype=np.float32)
        out_len = C.c_uint32(0)
        self._ck(self.lib.arroy_b200_rerank(self.h, _fp(query), qhdr[0], qhdr[1], _up(rows), rows.size, k, _up(out_rows), _fp(out_dist), C.byref(out_len)))
        return out_rows[:out_len.value].copy(), out_dist[:out_len.value].copy()

    def rerank_batch(self, queries, qhdr0, rows, offsets, k):
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        nq = queries.shape[0]
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        h0 = None if qhdr0 is None else np.ascontiguousarray(qhdr0, dtype=np.float32)
        out_rows = np.empty((nq, max(k, 1)), dtype=np.uint32)
        out_dist = np.empty((nq, max(k, 1)), dtype=np.float32)
        out_len = np.zeros(nq, dtype=np.uint32)
        self._ck(self.lib.arroy_b200_rerank_batch(self.h, nq, _fp(queries), _fp(h0), None, _up(rows), offsets.ctypes.data_as(_u64p), k,
                                                  _up(out_rows), _fp(out_dist), _up(out_len)))
        return out_rows, out_dist, out_len

    def rerank_shared(self, queries, qhdr0, rows, k):
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        nq = queries.shape[0]
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        h0 = None if qhdr0 is None else np.ascontiguousarray(qhdr0, dtype=np.float32)
        out_rows = np.empty((nq, max(k, 1)), dtype=np.uint32)
        out_dist = np.empty((nq, max(k, 1)), dtype=np.float32)
        out_len = np.zeros(nq, dtype=np.uint32)
        self._ck(self.lib.arroy_b200_rerank_shared(self.h, nq, _fp(queries), _fp(h0), _up(rows), rows.size, k, _up(out_rows), _fp(out_dist), _up(out_len)))
        return out_rows, out_dist, out_len

    # -- device-resident forest + batched search ----------------------------------------------------
    def load_forest(self, kind, left, right, normal_idx, normal_hdr0, desc_off, desc_len, normals, desc_rows, roots):
        a8 = np.ascontiguousarray(kind, dtype=np.uint8)
        u = lambda x: np.ascontiguousarray(x, dtype=np.uint32)
        left, right, normal_idx, desc_off, desc_len, desc_rows, roots = map(u, (left, right, normal_idx, desc_off, desc_len, desc_rows, roots))
        nh0 = np.ascontiguousarray(normal_hdr0, dtype=np.float32)
        normals = np.ascontiguousarray(normals, dtype=np.float32)
        self._ck(self.lib.arroy_b200_load_forest(self.h, a8.size, a8.ctypes.data_as(_u8p), _up(left), _up(right), _up(normal_idx), _fp(nh0), _up(desc_off), _up(desc_len),
                                                 normals.shape[0] if normals.ndim == 2 else 0, _fp(normals), desc_rows.size, _up(desc_rows), roots.size, _up(roots)))

    def search_batch(self, count, query_rows=None, queries=None, qhdr0=None, search_k=0):
        return self._search(count, query_rows, queries, qhdr0, search_k, None)

    def search_batch_filtered(self, count, filter_bits, query_rows=None, queries=None, qhdr0=None, search_k=0):
        """search_batch with one row filter for every query: filter_bits = ceil(n / 32) uint32 words, bit r = row r passes
        (row_bitmap builds it from row indices)."""
        bits = np.ascontiguousarray(filter_bits, dtype=np.uint32)
        if bits.size != (self.n + 31) // 32:
            raise ValueError("filter_bits must hold ceil(n / 32) = %d words" % ((self.n + 31) // 32))
        return self._search(count, query_rows, queries, qhdr0, search_k, bits)

    def search_batch_multi_filtered(self, count, filters, query_filter, query_rows=None, queries=None, qhdr0=None, search_k=0):
        """search_batch with one row filter per query: query q uses filters[query_filter[q]], a list of ascending, unique row
        indices. Several queries may share a filter; unused filters are allowed."""
        lists = [np.ascontiguousarray(f, dtype=np.uint32).ravel() for f in filters]
        offsets = np.zeros(len(lists) + 1, dtype=np.uint64)
        offsets[1:] = np.cumsum([f.size for f in lists])
        rows = np.concatenate(lists) if lists else np.zeros(0, np.uint32)
        qf = np.ascontiguousarray(query_filter, dtype=np.uint32)
        return self._search(count, query_rows, queries, qhdr0, search_k, None, (offsets, rows, qf))

    def _search(self, count, query_rows, queries, qhdr0, search_k, bits, multi=None):
        if query_rows is not None:
            query_rows = np.ascontiguousarray(query_rows, dtype=np.uint32)
            nq = query_rows.size
        else:
            queries = np.ascontiguousarray(queries, dtype=np.float32)
            nq = queries.shape[0]
        h0 = None if qhdr0 is None else np.ascontiguousarray(qhdr0, dtype=np.float32)
        out_rows = np.empty((nq, max(count, 1)), dtype=np.uint32)
        out_dist = np.empty((nq, max(count, 1)), dtype=np.float32)
        out_len = np.zeros(nq, dtype=np.uint32)
        status = np.zeros(nq, dtype=np.int32)
        st = status.ctypes.data_as(C.POINTER(C.c_int32))
        if multi is not None:
            offsets, rows, qf = multi
            if qf.size != nq:
                raise ValueError("query_filter must hold one filter index per query (%d)" % nq)
            self._ck(self.lib.arroy_b200_search_batch_multi_filtered(self.h, nq, _up(query_rows), _fp(queries), _fp(h0), count, search_k, offsets.size - 1,
                                                                     offsets.ctypes.data_as(_u64p), _up(rows), _up(qf), _up(out_rows), _fp(out_dist), _up(out_len), st))
        elif bits is None:
            self._ck(self.lib.arroy_b200_search_batch(self.h, nq, _up(query_rows), _fp(queries), _fp(h0), count, search_k, _up(out_rows), _fp(out_dist), _up(out_len), st))
        else:
            self._ck(self.lib.arroy_b200_search_batch_filtered(self.h, nq, _up(query_rows), _fp(queries), _fp(h0), count, search_k, _up(bits), _up(out_rows), _fp(out_dist),
                                                               _up(out_len), st))
        return out_rows, out_dist, out_len, status

    def search_stats(self):
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.arroy_b200_search_stats(self.h, out))
        return {"filtered_queries": int(out[0]), "shortcut_queries": int(out[1]), "failed_queries": int(out[2]), "nodes_popped": int(out[3])}

    def multi_filter_stats(self):
        out = (C.c_uint64 * 2)()
        self._ck(self.lib.arroy_b200_multi_filter_stats(self.h, out))
        return {"summary_passes": int(out[0]), "filters_summarised": int(out[1])}

    # -- helpers ---------------------------------------------------------------------------------
    def synth_device(self, seed, dim, row0, rows, centre, device_ptr):
        s = (C.c_uint8 * 32)(*bytes(seed))
        self._ck(self.lib.arroy_b200_synth_device(self.h, s, dim, row0, rows, centre, C.c_void_p(device_ptr)))

    def time_scan(self, normal, hdr, n_rows, rows=None, iters=5, flush_l2=True, variant=0):
        normal = np.ascontiguousarray(normal, dtype=np.float32)
        r = None if rows is None else np.ascontiguousarray(rows, dtype=np.uint32)
        ms = C.c_float(0)
        left = C.c_uint64(0)
        self._ck(self.lib.arroy_b200_time_scan(self.h, _fp(normal), hdr[0], hdr[1], _up(r), n_rows, variant, iters, 1 if flush_l2 else 0,
                                               C.byref(ms), C.byref(left)))
        return ms.value, left.value

    def build_breakdown(self):
        st = (C.c_double * 8)()
        self._ck(self.lib.arroy_b200_build_breakdown(self.h, st))
        keys = ["setup_ms", "graph_ms", "loop_ms", "d2h_ms", "encode_ms", "graph_launches", "schedules", "late_pool_slots"]
        return dict(zip(keys, list(st)))

    def counters(self):
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.arroy_b200_counters(self.h, out))
        return {"launches": out[0], "h2d_bytes": out[1], "d2h_bytes": out[2], "fused_rerank_batches": out[3] >> 32, "fused_rerank_fallbacks": out[3] & 0xffffffff}

    def plane_rerank_stats(self):
        """The plane pre-filter of host-placed indexes' batched re-ranks, since create (arroy_b200_plane_rerank_stats)."""
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.arroy_b200_plane_rerank_stats(self.h, out))
        return {"batches": out[0], "fallbacks": out[1], "rows_estimated": out[2], "rows_rescored": out[3]}

    def prefilter_scores(self, queries, rows, engine=0):
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        rows = np.ascontiguousarray(rows, dtype=np.uint32)
        out = np.empty((queries.shape[0], rows.size), dtype=np.float32)
        self._ck(self.lib.arroy_b200_prefilter_scores(self.h, queries.shape[0], _fp(queries), _up(rows), rows.size, engine, _fp(out)))
        return out

    def search_breakdown(self):
        out = (C.c_double * 8)()
        self._ck(self.lib.arroy_b200_search_breakdown(self.h, out))
        return dict(zip(["walk_ms", "sort_ms", "distance_ms", "topk_ms"], list(out)[:4]))

    def rerank_breakdown(self):
        out = (C.c_double * 8)()
        self._ck(self.lib.arroy_b200_rerank_breakdown(self.h, out))
        return dict(zip(["prep_ms", "score_gemm_ms", "select_ms", "rescore_ms", "topk_ms", "exact_dense_ms"], list(out)[:6]))

    def rerank_stats(self):
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.arroy_b200_rerank_stats(self.h, out))
        return {"prefilter_chunks": out[0], "fallback_chunks": out[1], "survivors": out[2], "queries": out[3]}

    def timer_start(self):
        self._ck(self.lib.arroy_b200_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float(0)
        self._ck(self.lib.arroy_b200_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def selftest_udiv(self, n_groups, seed=1):
        mism, fb = C.c_uint64(0), C.c_uint64(0)
        self._ck(self.lib.arroy_b200_selftest_udiv(self.h, n_groups, seed, C.byref(mism), C.byref(fb)))
        return int(mism.value), int(fb.value)

    def epochs(self):
        out = (C.c_uint64 * 2)()
        self._ck(self.lib.arroy_b200_epochs(self.h, out))
        return int(out[0]), int(out[1])

    def device_ptrs(self):
        out = (C.c_void_p * 3)()
        ld = C.c_uint32(0)
        self._ck(self.lib.arroy_b200_device_ptrs(self.h, out, C.byref(ld)))
        return [out[0], out[1], out[2]], ld.value


class Arena:
    """arroy_b200_arena: thread-safe append-only node sink (TmpNodes stand-in)."""

    def __init__(self):
        self.lib = load()
        self.h = C.c_void_p(self.lib.arroy_b200_arena_new())

    def clear(self):
        self.lib.arroy_b200_arena_clear(self.h)

    def stats(self):
        b = C.c_uint64(0)
        n = self.lib.arroy_b200_arena_stats(self.h, C.byref(b))
        return n, b.value

    def get(self, node_id):
        p = _u8p()
        ln = C.c_uint64(0)
        if self.lib.arroy_b200_arena_get(self.h, node_id, C.byref(p), C.byref(ln)) != 0:
            return None
        return C.string_at(p, ln.value)

    def __del__(self):
        try:
            self.lib.arroy_b200_arena_free(self.h)
        except Exception:
            pass


class Group:
    """Several GPUs of one node behind one handle (arroy_b200_create_group): in-library pipelined H2D + ncclBroadcast of
    the item buffer, trees sharded t mod n_dev, node ids as a single-device build."""

    def __init__(self, devices):
        self.lib = load()
        devs = (C.c_int32 * len(devices))(*devices)
        h = C.c_void_p()
        rc = self.lib.arroy_b200_create_group(len(devices), devs, C.byref(h))
        if rc != OK:
            raise ArroyB200Error(rc, "arroy_b200_create_group failed (device missing / NCCL not loadable)")
        self.h = h
        self.devices = list(devices)
        self.n = 0

    def _ck(self, rc):
        if rc != OK:
            raise ArroyB200Error(rc, self.lib.arroy_b200_group_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None):
            self.lib.arroy_b200_destroy_group(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def size(self):
        return self.lib.arroy_b200_group_size(self.h)

    def ctx(self, rank):
        """The member context of one device (owned by the group: do not close it)."""
        c = Context.__new__(Context)
        c.lib = self.lib
        c.h = C.c_void_p(self.lib.arroy_b200_group_ctx(self.h, rank))
        c.device = self.devices[rank]
        c.n, c.dim, c.metric = self.n, getattr(self, "dim", 0), getattr(self, "metric", None)
        c.close = lambda: None
        return c

    def stage_items_ptrs(self, metric, dim, ids, ptr_array):
        metric = METRICS[metric] if isinstance(metric, str) else metric
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        ptrs = np.ascontiguousarray(ptr_array, dtype=np.uint64)
        self._ck(self.lib.arroy_b200_group_stage_items(self.h, metric, dim, ids.size, _up(ids), ptrs.ctypes.data_as(C.POINTER(C.c_void_p))))
        self.n, self.dim, self.metric = ids.size, dim, metric

    def dot_preprocess(self):
        extra = np.empty(self.n, dtype=np.float32)
        norm = np.empty(self.n, dtype=np.float32)
        self._ck(self.lib.arroy_b200_group_dot_preprocess(self.h, _fp(extra), _fp(norm)))
        return extra, norm

    def build_trees(self, tree_seeds, root_ids, first_free_node_id, split_after=0, arena=None):
        """Returns {node id: bytes}, or the node count when an Arena collects the nodes."""
        n_trees = len(tree_seeds)
        seeds = (C.c_uint8 * (32 * max(n_trees, 1)))()
        for t, s in enumerate(tree_seeds):
            seeds[32 * t:32 * t + 32] = list(s)
        roots = np.ascontiguousarray(root_ids, dtype=np.uint32)
        n_nodes = C.c_uint64(0)
        if arena is not None:
            sink = C.cast(self.lib.arroy_b200_arena_sink, NODE_SINK)
            self._ck(self.lib.arroy_b200_group_build_trees(self.h, n_trees, C.cast(seeds, C.c_void_p), _up(roots), first_free_node_id, split_after,
                                                           C.cast(None, CANCEL_FN), None, sink, arena.h, C.byref(n_nodes)))
            return n_nodes.value
        out = {}
        import threading
        lock = threading.Lock()

        def sink(_arg, node_id, ptr, length):
            b = C.string_at(ptr, length)
            with lock:
                out[node_id] = b
            return 0

        cb = NODE_SINK(sink)
        self._ck(self.lib.arroy_b200_group_build_trees(self.h, n_trees, C.cast(seeds, C.c_void_p), _up(roots), first_free_node_id, split_after,
                                                       C.cast(None, CANCEL_FN), None, cb, None, C.byref(n_nodes)))
        return out

    def stage_breakdown(self):
        out = (C.c_double * 4)()
        self._ck(self.lib.arroy_b200_group_stage_breakdown(self.h, out))
        return {"total_ms": out[0], "tail_ms": out[1]}
