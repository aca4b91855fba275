"""Host-side mirror of pgvectorscale's `diskann` index-scan operator over the C ABI.

The reference's operator surface for this path is the four access-method callbacks
(`ambeginscan` / `amrescan` / `amgettuple` / `amendscan`,
pgvectorscale/src/access_method/scan.rs:309-476) plus the two query GUCs
(`diskann.query_search_list_size`, `diskann.query_rescore`, guc.rs:3-43).  `IndexScan`
keeps those names and argument meanings; `DiskAnnIndex.search_batch` is the batched form
(B independent scans, first k rows of each).  Everything here is a thin ctypes layer over
`libdiskann_b200.so` (include/diskann_b200.h): there is no Python or CPU implementation of
the search — if the CUDA library is missing or no device is visible the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from types import SimpleNamespace
from typing import Optional, Sequence

import numpy as np

from .build import LIB_PATH
from .snapshot import INVALID_NODE, Snapshot

INVALID_TID = 0xFFFFFFFFFFFFFFFF
QUERY_SEARCH_LIST_SIZE_DEFAULT = 100  # guc.rs:3
QUERY_RESCORE_DEFAULT = 50            # guc.rs:4


class DiskAnnError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"diskann_b200 error {code}: {message}")
        self.code = code


class _SnapshotDesc(C.Structure):
    _fields_ = [
        ("n", C.c_uint32), ("dim", C.c_uint32), ("dim_index", C.c_uint32), ("bits", C.c_uint32),
        ("words", C.c_uint32), ("R", C.c_uint32), ("distance_type", C.c_int32),
        ("has_labels", C.c_int32), ("count", C.c_uint64),
        ("mean", C.c_void_p), ("m2", C.c_void_p), ("codes", C.c_void_p), ("nbrs", C.c_void_p),
        ("heap_tid", C.c_void_p), ("vectors", C.c_void_p),
        ("start_default", C.c_uint32), ("n_start_labels", C.c_uint32),
        ("start_labels", C.c_void_p), ("start_label_nodes", C.c_void_p),
        ("label_off", C.c_void_p), ("labels", C.c_void_p),
    ]


class _BatchTiming(C.Structure):
    _fields_ = [("prepare_ms", C.c_float), ("search_ms", C.c_float), ("rerank_ms", C.c_float),
                ("resort_ms", C.c_float), ("total_ms", C.c_float), ("retries", C.c_uint32)]


class _SearchPlanInfo(C.Structure):
    _fields_ = [("kernel", C.c_uint32), ("slots_per_sm", C.c_uint32), ("grid", C.c_uint32), ("heap_smem", C.c_uint32),
                ("visited_cap", C.c_uint32), ("cand_cap", C.c_uint32), ("entry_bytes", C.c_uint32), ("bitmap", C.c_uint32),
                ("slot_hbm_bytes", C.c_uint64), ("smem_per_slot", C.c_uint32), ("retries", C.c_uint32)]


class _BuildStats(C.Structure):
    _fields_ = [("batches", C.c_uint32), ("search_ms", C.c_float), ("prune_ms", C.c_float), ("sort_ms", C.c_float),
                ("backlink_ms", C.c_float), ("total_ms", C.c_float), ("avg_degree", C.c_double)]


class _QueryStats(C.Structure):
    _fields_ = [("visits", C.c_uint32), ("d_quantized", C.c_uint32), ("candidates", C.c_uint32),
                ("d_full", C.c_uint32), ("stream_len", C.c_uint32), ("status", C.c_uint32)]


class _ScanWorkspace(C.Structure):
    _fields_ = [("mode", C.c_uint32), ("regrows", C.c_uint32), ("growths", C.c_uint32), ("reserved", C.c_uint32),
                ("device_bytes", C.c_uint64)]


# dann_query_params, one per query of a mixed batch
QUERY_PARAMS_DTYPE = np.dtype([("k", "<i4"), ("search_list_size", "<i4"), ("rescore", "<i4"), ("keyed", "<i4")])

STATS_DTYPE = np.dtype([("visits", "<u4"), ("d_quantized", "<u4"), ("candidates", "<u4"),
                        ("d_full", "<u4"), ("stream_len", "<u4"), ("status", "<u4")])

# every symbol include/diskann_b200.h declares
EXPORTS = [
    "dann_last_error", "dann_device_count", "dann_index_load", "dann_index_load_plain", "dann_index_free",
    "dann_coalescer_create", "dann_coalescer_search", "dann_coalescer_stats", "dann_coalescer_destroy",
    "dann_index_hbm_bytes", "dann_scan_begin", "dann_scan_rescan", "dann_scan_gettuple", "dann_scan_gettuple_many",
    "dann_coalescer_gettuple", "dann_scan_stats", "dann_scan_workspace", "dann_scan_end", "dann_search_batch", "dann_search_batch_device",
    "dann_scan_fetch",
    "dann_search_batch_mixed", "dann_search_batch_mixed_device", "dann_group_search_batch_mixed",
    "dann_prepare_queries", "dann_code_stride", "dann_sbq_distance", "dann_full_distance",
    "dann_kernel_launches", "dann_last_batch_timing",
    "dann_build_graph", "dann_index_download_nbrs", "dann_index_set_vectors", "dann_index_set_vectors_device",
    "dann_last_search_plan",
    "dann_group_create", "dann_group_size", "dann_group_replica", "dann_group_search_batch", "dann_group_free",
    "dann_shards_create", "dann_shards_count", "dann_shards_index", "dann_shards_search_batch", "dann_shards_free",
    "dann_shards_scan_begin", "dann_shards_scan_rescan", "dann_shards_scan_gettuple", "dann_shards_scan_stats",
    "dann_shards_scan_end",
    # relation-file reader (host only; mirror in pgreader.py)
    "dann_pg_relation_open", "dann_pg_relation_close", "dann_pg_relation_stat", "dann_pg_read_chain",
    "dann_pg_extract_sbq", "dann_pg_extract_plain", "dann_pg_snapshot_free", "dann_pg_heap_fetch_vectors",
]

_LIB = None


def load_library(path: Optional[str] = None):
    """dlopen the in-tree CUDA library; raises if it has not been built."""
    global _LIB
    if _LIB is not None and path is None:
        return _LIB
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise DiskAnnError(-3, f"{p} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback)")
    lib = C.CDLL(p)
    vp, u32p = C.c_void_p, C.POINTER(C.c_uint32)
    lib.dann_last_error.restype = C.c_char_p
    lib.dann_device_count.restype = C.c_int
    lib.dann_index_load.argtypes = [C.POINTER(_SnapshotDesc), C.c_int, C.POINTER(vp)]
    lib.dann_index_load_plain.argtypes = [C.POINTER(_SnapshotDesc), vp, C.c_int, C.POINTER(vp)]
    lib.dann_index_free.argtypes = [vp]
    lib.dann_index_free.restype = None
    lib.dann_index_hbm_bytes.argtypes = [vp]
    lib.dann_index_hbm_bytes.restype = C.c_uint64
    lib.dann_kernel_launches.argtypes = [vp]
    lib.dann_kernel_launches.restype = C.c_uint64
    lib.dann_code_stride.argtypes = [vp]
    lib.dann_code_stride.restype = C.c_uint32
    lib.dann_scan_begin.argtypes = [vp, C.POINTER(vp)]
    lib.dann_scan_rescan.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int]
    lib.dann_scan_gettuple.argtypes = [vp, u32p, C.POINTER(C.c_uint16), u32p, C.POINTER(C.c_float)]
    lib.dann_scan_fetch.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp]
    lib.dann_scan_gettuple_many.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp]
    lib.dann_scan_stats.argtypes = [vp, C.POINTER(_QueryStats)]
    lib.dann_scan_workspace.argtypes = [vp, C.POINTER(_ScanWorkspace)]
    lib.dann_scan_end.argtypes = [vp]
    lib.dann_scan_end.restype = None
    lib.dann_search_batch.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    lib.dann_search_batch_device.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                             vp, vp, vp, vp, vp]
    lib.dann_search_batch_mixed.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp]
    lib.dann_search_batch_mixed_device.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    lib.dann_group_search_batch_mixed.argtypes = [vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp]
    lib.dann_prepare_queries.argtypes = [vp, vp, C.c_int, vp, vp, vp]
    lib.dann_sbq_distance.argtypes = [vp, vp, vp, vp, C.c_size_t, vp, vp]
    lib.dann_full_distance.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp]
    lib.dann_last_batch_timing.argtypes = [vp, C.POINTER(_BatchTiming)]
    lib.dann_build_graph.argtypes = [vp, C.c_int, C.c_int, C.c_float, C.c_uint32, C.POINTER(_BuildStats)]
    lib.dann_index_download_nbrs.argtypes = [vp, vp]
    lib.dann_index_set_vectors.argtypes = [vp, vp]
    lib.dann_index_set_vectors_device.argtypes = [vp, vp]
    lib.dann_last_search_plan.argtypes = [vp, C.POINTER(_SearchPlanInfo)]
    lib.dann_group_create.argtypes = [C.POINTER(_SnapshotDesc), C.c_int, vp, C.POINTER(vp)]
    lib.dann_group_size.argtypes = [vp]
    lib.dann_group_replica.argtypes = [vp, C.c_int]
    lib.dann_group_replica.restype = vp
    lib.dann_group_search_batch.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    lib.dann_group_free.argtypes = [vp]
    lib.dann_group_free.restype = None
    lib.dann_shards_create.argtypes = [vp, C.c_int, vp, C.POINTER(vp)]
    lib.dann_shards_count.argtypes = [vp]
    lib.dann_shards_index.argtypes = [vp, C.c_int]
    lib.dann_shards_index.restype = vp
    lib.dann_shards_search_batch.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp]
    lib.dann_shards_free.argtypes = [vp]
    lib.dann_shards_free.restype = None
    lib.dann_shards_scan_begin.argtypes = [vp, C.POINTER(vp)]
    lib.dann_shards_scan_rescan.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int]
    lib.dann_shards_scan_gettuple.argtypes = [vp, u32p, C.POINTER(C.c_uint16), u32p, C.POINTER(C.c_float),
                                              C.POINTER(C.c_int32)]
    lib.dann_shards_scan_stats.argtypes = [vp, C.POINTER(_QueryStats)]
    lib.dann_shards_scan_end.argtypes = [vp]
    lib.dann_shards_scan_end.restype = None
    lib.dann_coalescer_create.argtypes = [vp, C.c_int, C.c_int, C.POINTER(vp)]
    lib.dann_coalescer_search.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    lib.dann_coalescer_gettuple.argtypes = [vp, vp, u32p, C.POINTER(C.c_uint16), u32p, C.POINTER(C.c_float)]
    lib.dann_coalescer_stats.argtypes = [vp, vp, vp, vp]
    lib.dann_coalescer_destroy.argtypes = [vp]
    lib.dann_coalescer_destroy.restype = None
    if path is None:
        _LIB = lib
    return lib


def _check(lib, rc: int):
    if rc < 0:
        raise DiskAnnError(rc, lib.dann_last_error().decode("utf-8", "replace"))
    return rc


def _np_ptr(a: Optional[np.ndarray]):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _dev_ptr(t):
    """torch CUDA tensor (or None / int) -> device pointer."""
    if t is None:
        return None
    if isinstance(t, int):
        return C.c_void_p(t)
    assert t.is_cuda and t.is_contiguous(), "device buffers must be contiguous CUDA tensors"
    return C.c_void_p(t.data_ptr())


def device_count() -> int:
    return int(load_library().dann_device_count())


def _make_desc(s: Snapshot):
    """dann_snapshot_desc over the snapshot's (contiguous) arrays; `keep` holds them alive for the call."""
    keep = []

    def arr(a, dt):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dt)
        keep.append(a)
        return C.c_void_p(a.ctypes.data)

    d = _SnapshotDesc()
    d.n, d.dim, d.dim_index, d.bits, d.words, d.R = s.n, s.dim, s.dim_index, s.bits, s.words, s.R
    d.distance_type = int(s.distance_type)
    d.has_labels = int(bool(s.has_labels))
    d.count = int(s.count)
    d.mean = arr(s.mean, np.float32)
    d.m2 = arr(s.m2, np.float32)
    d.codes = arr(s.codes, np.uint64)
    d.nbrs = arr(s.nbrs, np.uint32)
    d.heap_tid = arr(s.heap_tid, np.uint64)
    d.vectors = arr(s.vectors, np.float32)
    d.start_default = int(s.start_default)
    d.n_start_labels = 0 if s.start_labels is None else len(s.start_labels)
    d.start_labels = arr(s.start_labels, np.int16)
    d.start_label_nodes = arr(s.start_label_nodes, np.uint32)
    d.label_off = arr(s.label_off, np.uint32)
    d.labels = arr(s.labels, np.int16)
    return d, keep


class DiskAnnIndex:
    """One diskann index resident in the HBM of one GPU (dann_index_load)."""

    def __init__(self, snapshot: Snapshot, device: int = 0):
        self._lib = load_library()
        snapshot.validate()
        s = snapshot
        plain = int(getattr(s, "storage_type", 0) or 0) != 0
        d, keep = _make_desc(s)
        h = C.c_void_p()
        if plain:
            iv = np.ascontiguousarray(s.index_vectors, dtype=np.float32)
            assert iv.shape == (s.n, s.dim_index)
            keep.append(iv)
            _check(self._lib, self._lib.dann_index_load_plain(C.byref(d), C.c_void_p(iv.ctypes.data), int(device),
                                                              C.byref(h)))
        else:
            _check(self._lib, self._lib.dann_index_load(C.byref(d), int(device), C.byref(h)))
        self._h = h
        self._describe(s, device)

    def _describe(self, s, device: int):
        self.device = int(device)
        self.n, self.dim, self.dim_index = s.n, s.dim, s.dim_index
        self.bits, self.words, self.R = s.bits, s.words, s.R
        self.distance_type = int(s.distance_type)
        self.has_labels = bool(s.has_labels)

    @classmethod
    def _view(cls, owner, handle, snapshot, device: int) -> "DiskAnnIndex":
        """A non-owning DiskAnnIndex over an index handle that `owner` holds (and frees)."""
        v = cls.__new__(cls)
        v._lib, v._h, v._owner = owner._lib, C.c_void_p(handle), owner
        v._describe(snapshot, device)
        return v

    # -- lifetime -------------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            if getattr(self, "_owner", None) is None:
                self._lib.dann_index_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def hbm_bytes(self) -> int:
        return int(self._lib.dann_index_hbm_bytes(self._h))

    @property
    def kernel_launches(self) -> int:
        return int(self._lib.dann_kernel_launches(self._h))

    @property
    def code_stride(self) -> int:
        return int(self._lib.dann_code_stride(self._h))

    def last_search_plan(self) -> dict:
        t = _SearchPlanInfo()
        _check(self._lib, self._lib.dann_last_search_plan(self._h, C.byref(t)))
        return {k: int(getattr(t, k)) for k, _ in _SearchPlanInfo._fields_}

    def last_batch_timing(self) -> dict:
        t = _BatchTiming()
        _check(self._lib, self._lib.dann_last_batch_timing(self._h, C.byref(t)))
        return {k: getattr(t, k) for k, _ in _BatchTiming._fields_}

    # -- index construction (SURVEY §8f row 1; not the scan hot path) -----------------------------
    def build_graph(self, num_neighbors: int = 50, search_list_size: int = 100, max_alpha: float = 1.2,
                    max_batch: int = 1 << 20) -> dict:
        """GPU batch Vamana over the SBQ codes already in HBM (index loaded with R == 64 slots)."""
        st = _BuildStats()
        _check(self._lib, self._lib.dann_build_graph(self._h, int(num_neighbors), int(search_list_size),
                                                     float(max_alpha), int(max_batch), C.byref(st)))
        return {k: getattr(st, k) for k, _ in _BuildStats._fields_}

    def download_nbrs(self) -> np.ndarray:
        out = np.empty((self.n, self.R), np.uint32)
        _check(self._lib, self._lib.dann_index_download_nbrs(self._h, _np_ptr(out)))
        return out

    def set_vectors(self, vectors: np.ndarray):
        v = np.ascontiguousarray(vectors, dtype=np.float32)
        assert v.shape == (self.n, self.dim)
        _check(self._lib, self._lib.dann_index_set_vectors(self._h, _np_ptr(v)))

    def set_vectors_device(self, device_ptr: int):
        """Borrow [n][dim] f32 rows that already sit in this device's HBM (kept alive by the caller)."""
        _check(self._lib, self._lib.dann_index_set_vectors_device(self._h, C.c_void_p(int(device_ptr))))

    # -- scan operator ----------------------------------------------------------------
    def begin_scan(self) -> "IndexScan":
        """ambeginscan (scan.rs:309-333)."""
        return IndexScan(self)

    # -- batch ------------------------------------------------------------------------
    @staticmethod
    def _labels_csr(labels: Optional[Sequence[Optional[Sequence[int]]]], B: int, allow_unkeyed: bool = False):
        if labels is None:
            return None, None
        assert len(labels) == B
        off = np.zeros(B + 1, np.int32)
        vals = []
        for i, ls in enumerate(labels):
            if ls is None:
                if not allow_unkeyed:
                    raise ValueError("a batch is either all unkeyed (labels=None) or all keyed")
            else:
                vals.extend(int(x) for x in ls)
            off[i + 1] = len(vals)
        return np.asarray(vals, np.int16), off

    @staticmethod
    def _batch_params(B: int, labels, k, search_list_size, rescore):
        """None when every parameter is one int and no labels entry is None (the uniform dann_search_batch call), else
        the QUERY_PARAMS_DTYPE array [B] of dann_search_batch_mixed."""
        per_query = [np.ndim(x) > 0 for x in (k, search_list_size, rescore)]
        unkeyed = labels is not None and any(ls is None for ls in labels)
        if not any(per_query) and not unkeyed:
            return None
        p = np.empty(B, QUERY_PARAMS_DTYPE)
        for name, x in (("k", k), ("search_list_size", search_list_size), ("rescore", rescore)):
            a = np.asarray(x, dtype=np.int64)
            if a.ndim > 0 and a.shape != (B,):
                raise ValueError(f"{name} must be an int or a sequence of {B} ints")
            p[name] = a
        p["keyed"] = 0 if labels is None else [0 if ls is None else 1 for ls in labels]
        return p

    def search_batch(self, queries, labels=None, k=10, search_list_size=QUERY_SEARCH_LIST_SIZE_DEFAULT,
                     rescore=QUERY_RESCORE_DEFAULT, out=None):
        """B independent index scans from host buffers; returns the first k rows of each.

        queries: [B, dim] float32 (host).  labels: None, or one entry per query: a label list
        (`labels && ARRAY[...]`) or None (no scan key).  k, search_list_size and rescore are each an int or a
        sequence of B ints.  Returns dict(tid[B,kmax] u64 = (block<<16)|offset with INVALID_TID past count,
        dist[B,kmax] f32, count[B], stats[B]), kmax = the largest k.  One int each and no None label entry is
        dann_search_batch; anything else is dann_search_batch_mixed, with the same rows per query."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim != 2 or q.shape[1] != self.dim:
            raise ValueError(f"queries must be [B, {self.dim}]")
        B = q.shape[0]
        params = self._batch_params(B, labels, k, search_list_size, rescore)
        if params is not None:
            return self._search_batch_mixed(q, labels, params, out)
        lab, off = self._labels_csr(labels, B)
        if out is None:
            out = dict(tid=np.empty((B, k), np.uint64), dist=np.empty((B, k), np.float32),
                       count=np.empty(B, np.uint32), stats=np.empty(B, STATS_DTYPE))
        _check(self._lib, self._lib.dann_search_batch(
            self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and lab.size else None, _np_ptr(off),
            B, int(k), int(search_list_size), int(rescore),
            _np_ptr(out["tid"]), _np_ptr(out["dist"]), _np_ptr(out["count"]), _np_ptr(out["stats"])))
        return out

    def _search_batch_mixed(self, q, labels, params, out):
        B = q.shape[0]
        lab, off = self._labels_csr(labels, B, allow_unkeyed=True)
        kmax = int(params["k"].max()) if B else 0
        if out is None:
            out = dict(tid=np.empty((B, kmax), np.uint64), dist=np.empty((B, kmax), np.float32),
                       count=np.empty(B, np.uint32), stats=np.empty(B, STATS_DTYPE))
        _check(self._lib, self._lib.dann_search_batch_mixed(
            self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and lab.size else None, _np_ptr(off),
            _np_ptr(params), B, _np_ptr(out["tid"]), _np_ptr(out["dist"]), _np_ptr(out["count"]),
            _np_ptr(out["stats"])))
        return out

    def search_batch_mixed_device(self, d_queries, d_params, d_out_tid, d_out_dist=None, d_out_count=None,
                                  d_out_stats=None, d_labels=None, d_label_off=None, stream: int = 0):
        """dann_search_batch_mixed_device: every buffer in this device's HBM (torch CUDA tensors); d_params is
        [B] QUERY_PARAMS_DTYPE records (an int32 tensor [B, 4]), outputs [B, kmax]."""
        B = int(d_queries.shape[0])
        _check(self._lib, self._lib.dann_search_batch_mixed_device(
            self._h, _dev_ptr(d_queries), _dev_ptr(d_labels), _dev_ptr(d_label_off), _dev_ptr(d_params), B,
            _dev_ptr(d_out_tid), _dev_ptr(d_out_dist), _dev_ptr(d_out_count), _dev_ptr(d_out_stats),
            C.c_void_p(stream) if stream else None))

    def search_batch_ptrs(self, q_ptr: int, B: int, k: int, search_list_size: int, rescore: int,
                          tid_ptr: int, dist_ptr: int, count_ptr: int = 0, stats_ptr: int = 0,
                          labels_ptr: int = 0, label_off_ptr: int = 0):
        """dann_search_batch on raw HOST pointers (e.g. pinned torch tensors)."""
        vp = lambda x: C.c_void_p(x) if x else None
        _check(self._lib, self._lib.dann_search_batch(
            self._h, vp(q_ptr), vp(labels_ptr), vp(label_off_ptr), B, k, search_list_size, rescore,
            vp(tid_ptr), vp(dist_ptr), vp(count_ptr), vp(stats_ptr)))

    def search_batch_device(self, d_queries, k: int, search_list_size: int, rescore: int,
                            d_out_tid, d_out_dist=None, d_out_count=None, d_out_stats=None,
                            d_labels=None, d_label_off=None, stream: int = 0):
        """Same with every buffer already in this device's HBM (torch CUDA tensors)."""
        B = int(d_queries.shape[0])
        _check(self._lib, self._lib.dann_search_batch_device(
            self._h, _dev_ptr(d_queries), _dev_ptr(d_labels), _dev_ptr(d_label_off), B, int(k),
            int(search_list_size), int(rescore), _dev_ptr(d_out_tid), _dev_ptr(d_out_dist),
            _dev_ptr(d_out_count), _dev_ptr(d_out_stats), C.c_void_p(stream) if stream else None))

    # -- stand-alone kernels ------------------------------------------------------------
    def prepare_queries(self, d_queries, d_q_full, d_q_codes, stream: int = 0):
        _check(self._lib, self._lib.dann_prepare_queries(
            self._h, _dev_ptr(d_queries), int(d_queries.shape[0]), _dev_ptr(d_q_full),
            _dev_ptr(d_q_codes), C.c_void_p(stream) if stream else None))

    def sbq_distance(self, d_qcodes, d_pair_q, d_pair_node, d_out, stream: int = 0):
        _check(self._lib, self._lib.dann_sbq_distance(
            self._h, _dev_ptr(d_qcodes), _dev_ptr(d_pair_q), _dev_ptr(d_pair_node),
            int(d_pair_q.numel()), _dev_ptr(d_out), C.c_void_p(stream) if stream else None))

    def full_distance(self, d_q_full, d_nodes, d_out, stream: int = 0):
        B, m = int(d_nodes.shape[0]), int(d_nodes.shape[1])
        _check(self._lib, self._lib.dann_full_distance(
            self._h, _dev_ptr(d_q_full), _dev_ptr(d_nodes), B, m, _dev_ptr(d_out),
            C.c_void_p(stream) if stream else None))


class IndexScan:
    """ambeginscan / amrescan / amgettuple / amendscan (scan.rs:309-476) for one backend."""

    def __init__(self, index: DiskAnnIndex):
        self._index = index
        self._lib = index._lib
        h = C.c_void_p()
        _check(self._lib, self._lib.dann_scan_begin(index._h, C.byref(h)))
        self._h = h

    def rescan(self, query, labels: Optional[Sequence[int]] = None,
               search_list_size: int = QUERY_SEARCH_LIST_SIZE_DEFAULT,
               rescore: int = QUERY_RESCORE_DEFAULT):
        """amrescan: `ORDER BY embedding <op> query` (+ optional `labels && ARRAY[...]` key).
        query=None is a SQL NULL order-by argument; labels=None means no scan key."""
        q = None if query is None else np.ascontiguousarray(query, dtype=np.float32)
        if q is not None and q.shape != (self._index.dim,):
            raise ValueError(f"query must have {self._index.dim} dimensions")
        if labels is None:
            lab, nl = None, -1
        else:
            lab = np.ascontiguousarray(list(labels), dtype=np.int16)
            nl = int(lab.size)
        _check(self._lib, self._lib.dann_scan_rescan(
            self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and lab.size else None, nl,
            int(search_list_size), int(rescore)))

    def gettuple(self):
        """amgettuple: next row as (block, offset, node_id, distance) or None at end of scan."""
        b, o, n, d = C.c_uint32(), C.c_uint16(), C.c_uint32(), C.c_float()
        rc = _check(self._lib, self._lib.dann_scan_gettuple(self._h, C.byref(b), C.byref(o),
                                                            C.byref(n), C.byref(d)))
        if rc == 0:
            return None
        return int(b.value), int(o.value), int(n.value), float(d.value)

    def fetch(self, n: int):
        """The next n rows in one GPU step (dann_scan_fetch): exactly what n gettuple calls give.  Returns numpy arrays
        block, offset, node, dist of length r <= n (r < n only at end of scan) and a list of r dicts shaped like
        stats(): the scan's counters after each of those calls."""
        n = int(n)
        cap = max(n, 0)
        b = np.zeros(cap, np.uint32)
        o = np.zeros(cap, np.uint16)
        nd = np.zeros(cap, np.uint32)
        d = np.zeros(cap, np.float32)
        st = np.zeros(cap, STATS_DTYPE)
        r = _check(self._lib, self._lib.dann_scan_fetch(self._h, n, _np_ptr(b), _np_ptr(o), _np_ptr(nd), _np_ptr(d),
                                                         _np_ptr(st)))
        stats = [{k: int(row[k]) for k in STATS_DTYPE.names} for row in st[:r]]
        return b[:r], o[:r], nd[:r], d[:r], stats

    def stats(self) -> dict:
        st = _QueryStats()
        _check(self._lib, self._lib.dann_scan_stats(self._h, C.byref(st)))
        return {k: int(getattr(st, k)) for k, _ in _QueryStats._fields_}

    def workspace(self) -> dict:
        """What the scan holds (dann_scan_workspace): mode (0 = planned workspace, 1 = deep), regrows (replay regrows)
        and growths (in-place growths) since the last rescan, device_bytes held."""
        w = _ScanWorkspace()
        _check(self._lib, self._lib.dann_scan_workspace(self._h, C.byref(w)))
        return {k: int(getattr(w, k)) for k in ("mode", "regrows", "growths", "device_bytes")}

    def end(self):
        """amendscan."""
        if getattr(self, "_h", None):
            self._lib.dann_scan_end(self._h)
            self._h = None

    def __del__(self):
        try:
            self.end()
        except Exception:
            pass


def gettuple_many(scans: Sequence["IndexScan"]) -> list:
    """One amgettuple of each scan (all of one index) in one call (dann_scan_gettuple_many): the suspended searches
    resume together on the GPU.  Returns one entry per scan: the row as IndexScan.gettuple gives it, None at end of
    scan, or that scan's DiskAnnError (returned, not raised; its code is the scan's own, its message the call's last
    failure, dann_last_error).  Errors of the call itself raise."""
    scans = list(scans)
    n = len(scans)
    lib = scans[0]._lib if n else load_library()
    handles = (C.c_void_p * max(n, 1))(*[s._h for s in scans])
    rc = np.zeros(max(n, 1), np.int32)
    block = np.zeros(max(n, 1), np.uint32)
    offset = np.zeros(max(n, 1), np.uint16)
    node = np.zeros(max(n, 1), np.uint32)
    dist = np.zeros(max(n, 1), np.float32)
    _check(lib, lib.dann_scan_gettuple_many(handles, n, _np_ptr(rc), _np_ptr(block), _np_ptr(offset), _np_ptr(node),
                                            _np_ptr(dist)))
    err = lib.dann_last_error().decode("utf-8", "replace")
    out = []
    for i in range(n):
        if rc[i] < 0:
            out.append(DiskAnnError(int(rc[i]), err))
        elif rc[i] == 0:
            out.append(None)
        else:
            out.append((int(block[i]), int(offset[i]), int(node[i]), float(dist[i])))
    return out


class IndexGroup:
    """dann_group: one replica of the index per GPU inside this process; a batch is split into contiguous slices, every
    device runs the whole hot path on its slice, rows come back in query order (SURVEY.md §8b / §8e)."""

    def __init__(self, snapshot: Snapshot, devices: Optional[Sequence[int]] = None, ndev: Optional[int] = None):
        self._lib = load_library()
        snapshot.validate()
        d, keep = _make_desc(snapshot)
        devs = None if devices is None else np.ascontiguousarray(list(devices), dtype=np.int32)
        n = len(devs) if devs is not None else int(ndev if ndev is not None else device_count())
        h = C.c_void_p()
        _check(self._lib, self._lib.dann_group_create(C.byref(d), n, _np_ptr(devs), C.byref(h)))
        self._h = h
        self.dim = snapshot.dim
        self.size = int(self._lib.dann_group_size(h))
        del keep

    def search_batch(self, queries, labels=None, k=10, search_list_size=QUERY_SEARCH_LIST_SIZE_DEFAULT,
                     rescore=QUERY_RESCORE_DEFAULT) -> dict:
        """As DiskAnnIndex.search_batch: k, search_list_size and rescore may be per-query sequences and labels
        entries None (dann_group_search_batch_mixed)."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        B = q.shape[0]
        params = DiskAnnIndex._batch_params(B, labels, k, search_list_size, rescore)
        if params is not None:
            lab, off = DiskAnnIndex._labels_csr(labels, B, allow_unkeyed=True)
            kmax = int(params["k"].max()) if B else 0
            out = dict(tid=np.empty((B, kmax), np.uint64), dist=np.empty((B, kmax), np.float32),
                       count=np.empty(B, np.uint32), stats=np.empty(B, STATS_DTYPE))
            _check(self._lib, self._lib.dann_group_search_batch_mixed(
                self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and lab.size else None, _np_ptr(off),
                _np_ptr(params), B, _np_ptr(out["tid"]), _np_ptr(out["dist"]), _np_ptr(out["count"]),
                _np_ptr(out["stats"])))
            return out
        lab, off = DiskAnnIndex._labels_csr(labels, B)
        out = dict(tid=np.empty((B, k), np.uint64), dist=np.empty((B, k), np.float32),
                   count=np.empty(B, np.uint32), stats=np.empty(B, STATS_DTYPE))
        _check(self._lib, self._lib.dann_group_search_batch(
            self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and lab.size else None, _np_ptr(off), B, int(k),
            int(search_list_size), int(rescore), _np_ptr(out["tid"]), _np_ptr(out["dist"]), _np_ptr(out["count"]),
            _np_ptr(out["stats"])))
        return out

    def close(self):
        if getattr(self, "_h", None):
            self._lib.dann_group_free(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_GEOMETRY = ("n", "dim", "dim_index", "bits", "words", "R", "distance_type", "has_labels")


class ShardedIndex:
    """dann_shards: a table split into shards, one independent index per shard (its own graph, means and start nodes),
    on one or several GPUs.  search_batch runs every shard on all queries and merges their rows on the device of shard
    0: k times the head with the smallest (f32::total_cmp key of its distance, shard index) among the shards' lists."""

    def __init__(self, snapshots: Sequence[Snapshot], devices: Optional[Sequence[int]] = None):
        self._lib = load_library()
        snaps = list(snapshots)
        descs, keep = [], []
        for s in snaps:
            s.validate()
            d, kp = _make_desc(s)
            descs.append(d)
            keep.append(kp)
        arr = (C.POINTER(_SnapshotDesc) * max(len(descs), 1))(*[C.pointer(d) for d in descs])
        devs = None if devices is None else np.ascontiguousarray(list(devices), dtype=np.int32)
        h = C.c_void_p()
        _check(self._lib, self._lib.dann_shards_create(C.cast(arr, C.c_void_p), len(descs), _np_ptr(devs), C.byref(h)))
        self._h = h
        self.dim = snaps[0].dim
        self.count = int(self._lib.dann_shards_count(h))
        self.devices = [int(x) for x in devs] if devs is not None else list(range(self.count))
        # each shard's geometry for its view (not the arrays: the index has its own copy in HBM)
        self._geom = [SimpleNamespace(**{f: getattr(s, f) for f in _GEOMETRY}) for s in snaps]
        del keep

    def shard(self, i: int) -> DiskAnnIndex:
        """Shard i as a non-owning DiskAnnIndex (build_graph, set_vectors, set_vectors_device, last_batch_timing ...);
        valid while this ShardedIndex is open."""
        if not 0 <= i < self.count:
            raise IndexError(f"shard {i} of {self.count}")
        h = self._lib.dann_shards_index(self._h, int(i))
        return DiskAnnIndex._view(self, h, self._geom[i], self.devices[i])

    def begin_scan(self) -> "ShardedScan":
        """ambeginscan over every shard: one streaming scan whose rows are the shards' scans merged."""
        return ShardedScan(self)

    def search_batch(self, queries, labels=None, k: int = 10, search_list_size: int = QUERY_SEARCH_LIST_SIZE_DEFAULT,
                     rescore: int = QUERY_RESCORE_DEFAULT) -> dict:
        """Merged first k rows of B queries over every shard: dict(tid[B,k], dist[B,k], shard[B,k] i32 (-1 past count),
        count[B], stats[nshards, B])."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim != 2 or q.shape[1] != self.dim:
            raise ValueError(f"queries must be [B, {self.dim}]")
        B = q.shape[0]
        lab, off = DiskAnnIndex._labels_csr(labels, B)
        out = dict(tid=np.empty((B, k), np.uint64), dist=np.empty((B, k), np.float32),
                   shard=np.empty((B, k), np.int32), count=np.empty(B, np.uint32),
                   stats=np.empty((self.count, B), STATS_DTYPE))
        _check(self._lib, self._lib.dann_shards_search_batch(
            self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and lab.size else None, _np_ptr(off), B, int(k),
            int(search_list_size), int(rescore), _np_ptr(out["tid"]), _np_ptr(out["dist"]), _np_ptr(out["shard"]),
            _np_ptr(out["count"]), _np_ptr(out["stats"])))
        return out

    def close(self):
        if getattr(self, "_h", None):
            self._lib.dann_shards_free(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShardedScan:
    """amrescan / amgettuple / amendscan over a sharded table (dann_shards_scan_*): one IndexScan per shard, merged one
    row at a time by the rule of ShardedIndex.search_batch, so its first k rows are the batch's k rows.  The first
    gettuple after a rescan steps every shard (the shards of one device in one launch round); each later call steps the
    shard whose row the previous call returned."""

    def __init__(self, index: ShardedIndex):
        self._index = index
        self._lib = index._lib
        h = C.c_void_p()
        _check(self._lib, self._lib.dann_shards_scan_begin(index._h, C.byref(h)))
        self._h = h

    def rescan(self, query, labels: Optional[Sequence[int]] = None,
               search_list_size: int = QUERY_SEARCH_LIST_SIZE_DEFAULT,
               rescore: int = QUERY_RESCORE_DEFAULT):
        """amrescan on every shard, as IndexScan.rescan; rescore must be > 0."""
        q = None if query is None else np.ascontiguousarray(query, dtype=np.float32)
        if q is not None and q.shape != (self._index.dim,):
            raise ValueError(f"query must have {self._index.dim} dimensions")
        if labels is None:
            lab, nl = None, -1
        else:
            lab = np.ascontiguousarray(list(labels), dtype=np.int16)
            nl = int(lab.size)
        _check(self._lib, self._lib.dann_shards_scan_rescan(
            self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and lab.size else None, nl,
            int(search_list_size), int(rescore)))

    def gettuple(self):
        """amgettuple: next merged row as (block, offset, node_id, distance, shard) or None at end of scan; node_id is
        local to its shard."""
        b, o, n, d, s = C.c_uint32(), C.c_uint16(), C.c_uint32(), C.c_float(), C.c_int32()
        rc = _check(self._lib, self._lib.dann_shards_scan_gettuple(self._h, C.byref(b), C.byref(o), C.byref(n),
                                                                   C.byref(d), C.byref(s)))
        if rc == 0:
            return None
        return int(b.value), int(o.value), int(n.value), float(d.value), int(s.value)

    def stats(self) -> list:
        """One dict per shard: that shard's scan counters (IndexScan.stats)."""
        st = (_QueryStats * self._index.count)()
        _check(self._lib, self._lib.dann_shards_scan_stats(self._h, st))
        return [{k: int(getattr(x, k)) for k, _ in _QueryStats._fields_} for x in st]

    def end(self):
        """amendscan."""
        if getattr(self, "_h", None):
            self._lib.dann_shards_scan_end(self._h)
            self._h = None

    def __del__(self):
        try:
            self.end()
        except Exception:
            pass


class Coalescer:
    """dann_coalescer: single-query callers (one thread per connected backend in a sidecar) coalesced into batch calls
    (SURVEY.md §8f row 4).  search() blocks and may be called from many threads at once (ctypes drops the GIL)."""

    def __init__(self, index: DiskAnnIndex, max_batch: int = 256, max_wait_us: int = 200):
        self._lib = index._lib
        self._index = index
        h = C.c_void_p()
        _check(self._lib, self._lib.dann_coalescer_create(index._h, int(max_batch), int(max_wait_us), C.byref(h)))
        self._h = h

    def search(self, query, labels: Optional[Sequence[int]] = None, k: int = 10,
               search_list_size: int = QUERY_SEARCH_LIST_SIZE_DEFAULT, rescore: int = QUERY_RESCORE_DEFAULT) -> dict:
        q = np.ascontiguousarray(query, dtype=np.float32)
        if q.shape != (self._index.dim,):
            raise ValueError(f"query must have {self._index.dim} dimensions")
        lab = None if labels is None else np.asarray(list(labels), dtype=np.int16)
        tid = np.full(k, 0xFFFFFFFFFFFFFFFF, np.uint64)
        dist = np.zeros(k, np.float32)
        count = C.c_uint32()
        st = _QueryStats()
        _check(self._lib, self._lib.dann_coalescer_search(
            self._h, _np_ptr(q), _np_ptr(lab) if lab is not None and len(lab) else None, -1 if lab is None else len(lab),
            int(k), int(search_list_size), int(rescore), _np_ptr(tid), _np_ptr(dist), C.byref(count), C.byref(st)))
        return dict(tid=tid, dist=dist, count=int(count.value),
                    stats={f: int(getattr(st, f)) for f, _ in _QueryStats._fields_})

    def gettuple(self, scan: "IndexScan"):
        """IndexScan.gettuple through the dispatcher: gettuple calls of many threads (any scans of this index) that
        arrive together become one dann_scan_gettuple_many.  Blocks; returns what scan.gettuple() would."""
        b, o, n, d = C.c_uint32(), C.c_uint16(), C.c_uint32(), C.c_float()
        rc = _check(self._lib, self._lib.dann_coalescer_gettuple(self._h, scan._h, C.byref(b), C.byref(o), C.byref(n),
                                                                 C.byref(d)))
        if rc == 0:
            return None
        return int(b.value), int(o.value), int(n.value), float(d.value)

    def stats(self) -> dict:
        """batches / queries / largest_batch count search and gettuple dispatches alike."""
        b, q, m = C.c_uint64(), C.c_uint64(), C.c_uint64()
        _check(self._lib, self._lib.dann_coalescer_stats(self._h, C.byref(b), C.byref(q), C.byref(m)))
        return dict(batches=int(b.value), queries=int(q.value), largest_batch=int(m.value))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.dann_coalescer_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
