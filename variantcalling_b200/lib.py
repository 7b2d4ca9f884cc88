"""ctypes binding of ``libugvc_b200.so`` (C ABI: ``include/ugvc_b200.h``).

There is no CPU fallback: importing the library needs the built shared object,
and creating a :class:`Context` needs a CUDA device -- both fail loudly.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("UGVC_LIB_PATH") or os.path.join(_HERE, "libugvc_b200.so")  # env: profiling builds

UGVC_OK, UGVC_E_CUDA, UGVC_E_ARG, UGVC_E_PLAN, UGVC_E_DATA, UGVC_E_IO, UGVC_E_STATE = 0, -1, -2, -3, -4, -5, -6
UGVC_E_FALLBACK = -7  # ugvc_filter_bgzf: a record needs the general host writer
FILE_OVERWRITE_QUAL, FILE_BLACKLIST_CG = 1, 2
DEF_CHUNK = 57344     # uncompressed bytes per BGZF block written by the device encoder


class UgvcError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"[ugvc {code}] {message}")
        self.code = code
        self.message = message


class UgvcDataError(UgvcError, AssertionError):
    """The reference pipeline would raise on this input (null feature, unknown
    category, ragged tuple ...); mirrors ``_validate_data``'s AssertionError."""


RECINFO_DTYPE = np.dtype([("pos", "<i4"), ("qual_off", "<u2"), ("filter_off", "<u2"), ("info_off", "<u2"),
                          ("format_off", "<u2"), ("flags", "<u4")])


class FileEdits(C.Structure):
    """ugvc_file_edits (include/ugvc_b200.h)."""
    _fields_ = [("with_model", C.c_int), ("recalibrate_genotype", C.c_int), ("n_blacklists", C.c_int),
                ("blacklist_pos", C.c_void_p), ("blacklist_pos_off", C.c_void_p), ("blacklist_names", C.c_void_p),
                ("blacklist_name_off", C.c_void_p), ("out_end", C.c_void_p), ("n_blacklisted", C.c_int64)]


class AfrParams(C.Structure):
    """ugvc_afr_params (include/ugvc_b200.h)."""
    _fields_ = [("af_ratio_threshold", C.c_double), ("af_ratio_threshold_h_indels", C.c_double), ("t_vaf_threshold", C.c_double),
                ("new_filter", C.c_char_p), ("new_filter_len", C.c_int32), ("variant_type_kind", C.c_int32),
                ("vaf_kind", C.c_int32), ("vaf_integer", C.c_int32), ("bg_vaf_kind", C.c_int32), ("bg_vaf_integer", C.c_int32)]


AFR_KIND_NONE, AFR_KIND_SCALAR, AFR_KIND_TUPLE = 0, 1, 2
AFR_E_LITERAL, AFR_E_TYPE = 1, 2
AFR_FAILED, AFR_REWRITTEN, AFR_NEW_CONTIG = 1, 2, 4
AFR_MAX_FILTER_BYTES = 63


class BsnParams(C.Structure):
    """ugvc_bsn_params (include/ugvc_b200.h)."""
    _fields_ = [("min_query_hmer_size", C.c_int32), ("min_distance_from_edge", C.c_int32), ("min_initial_qual", C.c_double),
                ("min_tumor_vaf", C.c_double), ("max_normal_vaf", C.c_double), ("min_normal_depth", C.c_double),
                ("qual_text", C.c_char_p), ("qual_len", C.c_int32), ("ad_kind", C.c_int32), ("ad_integer", C.c_int32),
                ("dp_kind", C.c_int32), ("dp_integer", C.c_int32), ("bg_ad_kind", C.c_int32), ("bg_ad_integer", C.c_int32),
                ("bg_dp_kind", C.c_int32), ("bg_dp_integer", C.c_int32)]


BSN_KIND_NONE, BSN_KIND_SCALAR, BSN_KIND_TUPLE = 0, 1, 2
BSN_E_LITERAL, BSN_E_TYPE, BSN_E_ZERO_DIVISION, BSN_E_KEY, BSN_E_FETCH = 1, 2, 3, 4, 5
BSN_RESCUED, BSN_NEW_CONTIG = 1, 4
BSN_MAX_QUAL_BYTES = 31


class HcrParams(C.Structure):
    """ugvc_hcr_params (include/ugvc_b200.h)."""
    _fields_ = [("gq_threshold", C.c_int64), ("gt", C.c_int32), ("merge", C.c_int32), ("info_end", C.c_int32),
                ("gq_kind", C.c_int32), ("gq_integer", C.c_int32)]


HCR_GQ_STRING, HCR_GQ_SCALAR, HCR_GQ_TUPLE = 0, 1, 2
HCR_E_LITERAL, HCR_E_TYPE, HCR_E_KEY, HCR_E_UNSORTED = 1, 2, 3, 4
HCR_SELECTED, HCR_GQ_ERROR, HCR_NEW_CONTIG, HCR_RESET, HCR_KEPT, HCR_LINE = 1, 2, 4, 8, 16, 32


class Counts(C.Structure):
    _fields_ = [("n_records", C.c_int64), ("n_low_score", C.c_int64), ("n_pass", C.c_int64), ("n_cg", C.c_int64)]


_vp, _sz, _i64p = C.c_void_p, C.c_size_t, C.POINTER(C.c_int64)

# name -> (restype, argtypes); every symbol declared in include/ugvc_b200.h
SIGNATURES = {
    "ugvc_init": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "ugvc_free": (None, [_vp]),
    "ugvc_last_error": (C.c_char_p, [_vp]),
    "ugvc_version": (C.c_int, []),
    "ugvc_load_plan": (C.c_int, [_vp, _vp, _sz]),
    "ugvc_plan_info": (C.c_int, [_vp, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "ugvc_reserve": (C.c_int, [_vp, _sz, _sz, C.c_int]),
    "ugvc_set_key_order": (C.c_int, [_vp, C.c_char_p, C.c_char_p]),
    "ugvc_debug_slow_records": (C.c_int64, [_vp, C.c_int]),
    "ugvc_filter_batch": (C.c_int, [_vp, _vp, _sz, C.c_double, _vp, _vp, _vp, _vp, _vp, _sz, _i64p]),
    "ugvc_submit_batch": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_double]),
    "ugvc_collect_batch": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp, _vp, _vp, _sz, _i64p]),
    "ugvc_filter_device": (C.c_int, [_vp, _vp, _sz, C.c_double, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "ugvc_device_status": (C.c_int, [_vp, _vp]),
    "ugvc_filter_device_lane": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_double, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "ugvc_device_status_lane": (C.c_int, [_vp, C.c_int, _vp]),
    "ugvc_nccl_unique_id": (C.c_int, [_vp]),
    "ugvc_nccl_comm_init": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.POINTER(_vp)]),
    "ugvc_nccl_comm_destroy": (C.c_int, [_vp]),
    "ugvc_counts_allreduce": (C.c_int, [_vp, _vp, _vp, _vp]),
    "ugvc_bind_thread": (C.c_int, [_vp]),
    "ugvc_host_alloc": (C.c_int, [C.POINTER(_vp), _sz]),
    "ugvc_host_free": (C.c_int, [_vp]),
    "ugvc_counts_reset": (C.c_int, [_vp]),
    "ugvc_counts_get": (C.c_int, [_vp, C.POINTER(Counts)]),
    "ugvc_counts_device_ptr": (C.c_int, [_vp, C.POINTER(_vp)]),
    "ugvc_debug_raw": (C.c_int, [_vp, C.c_int, _vp, _sz]),
    "ugvc_debug_features": (C.c_int, [_vp, C.c_int, _vp, _sz]),
    "ugvc_last_data_error": (C.c_int, [_vp, _i64p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "ugvc_launch_count": (C.c_int64, [_vp]),
    "ugvc_enable_stage_timing": (C.c_int, [_vp, C.c_int]),
    "ugvc_stage_ms": (C.c_int, [_vp, C.POINTER(C.c_float), _i64p]),
    "ugvc_synth_device": (C.c_int, [_vp, C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_int, _vp, _sz,
                                    C.POINTER(_sz), _vp]),
    "ugvc_synth_header": (C.c_int64, [C.c_int, C.c_char_p, _sz]),
    "ugvc_bgzf_inflate_file": (C.c_int, [C.c_char_p, C.c_uint64, C.c_uint64, _vp, _sz, C.POINTER(_sz), C.c_int]),
    "ugvc_bgzf_uncompressed_size": (C.c_int64, [C.c_char_p]),
    "ugvc_bgzf_deflate_to_file": (C.c_int, [C.c_char_p, C.c_char_p, _vp, _sz, C.c_int, C.c_int, C.c_int,
                                            C.POINTER(C.c_uint64), _vp, _sz, C.POINTER(_sz)]),
    "ugvc_count_byte": (C.c_int64, [_vp, _sz, C.c_int, C.c_int]),
    "ugvc_info_end": (C.c_int64, [_vp, _vp, _vp, C.c_int64, _vp, C.c_int]),
    "ugvc_splice_records": (C.c_int64, [_vp, _vp, _vp, _vp, _vp, C.c_int64, C.c_int, C.c_int, _vp, _vp, _vp,
                                        _vp, C.c_int, _vp, _sz, _vp, C.c_int]),
    "ugvc_submit_bgzf": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_double]),
    "ugvc_bgzf_inflate_device": (C.c_int, [_vp, _vp, _sz, _vp, _sz, C.POINTER(_sz)]),
    "ugvc_predict_features": (C.c_int, [_vp, _vp, _sz, _sz, C.c_double, _vp, _vp, _vp]),
    "ugvc_enable_phreds": (C.c_int, [_vp, C.c_int]),
    "ugvc_collect_phreds": (C.c_int, [_vp, C.c_int, _vp, _sz]),
    "ugvc_conc_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "ugvc_conc_free": (None, [_vp]),
    "ugvc_conc_last_error": (C.c_char_p, [_vp]),
    "ugvc_conc_launch_count": (C.c_longlong, [_vp]),
    # out_counts: int64[9][8] (UGVC_CONC_GROUPS x UGVC_CONC_COUNTERS, the last two: NaN / inf scores of called records)
    "ugvc_conc_run": (C.c_int, [_vp, C.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp]),
    "ugvc_conc_classify": (C.c_int, [_vp, C.c_int64, _vp, _vp, _vp, _vp, _vp]),
    "ugvc_conc_curve": (C.c_int, [_vp, C.c_int, _vp, _vp, _vp, _sz]),
    "ugvc_conc_annot_add_contig": (C.c_int, [_vp, _vp, C.c_int64, _vp]),
    "ugvc_conc_annot_clear": (C.c_int, [_vp]),
    "ugvc_conc_annotate": (C.c_int, [_vp, C.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, C.c_char_p, C.c_int,
                                     C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ugvc_conc_annot_error": (C.c_int, [_vp, _vp, _vp]),
    "ugvc_conc_annot_kernel_ms": (C.c_double, [_vp]),
    "ugvc_ma_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "ugvc_ma_free": (None, [_vp]),
    "ugvc_ma_last_error": (C.c_char_p, [_vp]),
    "ugvc_ma_launch_count": (C.c_longlong, [_vp]),
    "ugvc_ma_set_rules": (C.c_int, [_vp, _vp, _sz]),
    "ugvc_ma_build": (C.c_int, [_vp, _vp, _sz, _vp, _vp, C.c_int64, _vp, _sz, _i64p]),
    "ugvc_ma_data_error": (C.c_int, [_vp, _i64p, C.POINTER(C.c_int32)]),
    "ugvc_ma_fetch": (C.c_int, [_vp, _vp, _sz, _vp, _vp, _vp, _sz]),
    "ugvc_ma_merge": (C.c_int, [_vp, _vp, C.c_int64, C.c_int, _vp, C.c_int]),
    "ugvc_tbi_summary": (C.c_int, [_vp, C.c_size_t, C.c_int32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ugvc_test_deflate_block": (C.c_int64, [_vp, C.c_uint32, _vp]),
    "ugvc_test_deflate_block_lanes": (C.c_int64, [_vp, C.c_uint32, _vp]),
    "ugvc_test_device_sigmoid": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp]),
    "ugvc_test_k3_config": (C.c_int, [_vp, _vp]),
    "ugvc_test_format_g": (C.c_int, [_vp, _vp, C.c_int64, _vp]),
    "ugvc_test_device_deflate": (C.c_int, [_vp, _vp, _sz, C.c_int, _vp, _sz, _vp, _sz, C.POINTER(_sz), C.POINTER(_sz)]),
    "ugvc_test_device_inflate": (C.c_int, [_vp, _vp, _sz, C.c_int, _vp, _sz, C.POINTER(_sz), _vp, _sz, C.POINTER(_sz)]),
    "ugvc_bgzf_range_info": (C.c_int, [C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]),
    "ugvc_filter_bgzf": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_uint32, C.c_uint64, C.c_double, C.c_int, _vp, _sz, C.POINTER(_sz),
                                   _vp, _sz, C.POINTER(_sz), _vp, _vp, _vp, _sz, C.POINTER(C.c_int64)]),
    "ugvc_filter_bgzf_edits": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_uint32, C.c_uint64, C.c_double, C.c_int, C.POINTER(FileEdits),
                                         _vp, _sz, C.POINTER(_sz), _vp, _sz, C.POINTER(_sz), _vp, _vp, _vp, _sz,
                                         C.POINTER(C.c_int64)]),
    "ugvc_test_write_records": (C.c_int64, [_vp, _vp, _sz, _vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_int, C.c_int,
                                            C.POINTER(FileEdits), _vp, _sz, _vp]),
    "ugvc_filter_bgzf_stage_ms": (C.c_int, [_vp, C.c_int, _vp]),
    "ugvc_filter_bgzf_split": (C.c_int, [_vp, _vp, _vp, C.c_int, _vp, _sz, C.c_uint32, C.c_uint64, _vp, _sz, C.c_double, C.c_int,
                                         C.POINTER(FileEdits), _vp, _sz, C.POINTER(_sz), _vp, _sz, C.POINTER(_sz), _vp, _vp, _vp,
                                         _sz, C.POINTER(C.c_int64), _vp]),
    "ugvc_filter_bgzf_split_stage_ms": (C.c_int, [_vp, C.c_int, _vp]),
    "ugvc_test_ma_score": (C.c_int, [_vp, _vp, C.c_int64, C.c_int, C.c_double, _vp, _vp, _vp]),
    "ugvc_filter_bgzf_first_records": (C.c_int, [_vp, C.c_int, _vp, C.c_int, _vp]),
    "ugvc_test_parse_float": (C.c_int, [C.c_char_p, C.POINTER(C.c_float), C.POINTER(C.c_double),
                                        C.POINTER(C.c_int)]),
    "ugvc_afr_bgzf": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_uint32, C.c_uint64, C.c_int, C.POINTER(AfrParams), _vp, _sz,
                                C.POINTER(_sz), _vp, _sz, C.POINTER(_sz), _vp, _vp, _vp, _vp, _sz, _i64p, _i64p]),
    "ugvc_afr_error": (C.c_int, [_vp, C.c_int, _i64p, C.POINTER(C.c_int32)]),
    "ugvc_afr_stage_ms": (C.c_int, [_vp, C.c_int, _vp]),
    "ugvc_test_afr": (C.c_int64, [_vp, _sz, _vp, C.c_int64, C.POINTER(AfrParams), _vp, _sz, _vp, _vp, _vp, _i64p, _i64p,
                                  C.POINTER(C.c_int32)]),
    "ugvc_bsn_add_contig": (C.c_int, [_vp, C.c_char_p, _vp, C.c_int64]),
    "ugvc_bsn_clear_contigs": (C.c_int, [_vp]),
    "ugvc_bsn_bgzf": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_uint32, C.c_uint64, C.c_int, C.POINTER(BsnParams), _vp, _sz,
                                C.POINTER(_sz), _vp, _sz, C.POINTER(_sz), _vp, _vp, _vp, _vp, _vp, _vp, _sz, _i64p, _i64p]),
    "ugvc_bsn_error": (C.c_int, [_vp, C.c_int, _i64p, C.POINTER(C.c_int32)]),
    "ugvc_bsn_stage_ms": (C.c_int, [_vp, C.c_int, _vp]),
    "ugvc_test_bsn": (C.c_int64, [_vp, _sz, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_int32, C.POINTER(BsnParams), _vp, _sz,
                                  _vp, _vp, _vp, _vp, _i64p, _i64p, C.POINTER(C.c_int32)]),
    "ugvc_hcr_scan": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_uint32, C.c_uint64, C.POINTER(HcrParams), _sz, _i64p, _vp, _vp]),
    "ugvc_hcr_emit": (C.c_int, [_vp, C.c_int, C.POINTER(HcrParams), C.c_int, C.c_int64, _vp, _sz, C.POINTER(_sz), _vp]),
    "ugvc_hcr_error": (C.c_int, [_vp, C.c_int, _i64p, C.POINTER(C.c_int32)]),
    "ugvc_hcr_stage_ms": (C.c_int, [_vp, C.c_int, _vp]),
    "ugvc_test_hcr": (C.c_int64, [_vp, _sz, _vp, C.c_int64, C.POINTER(HcrParams), C.c_int, C.c_int64, C.c_int64, _vp, _sz,
                                  _vp, _vp, _i64p, C.POINTER(C.c_int32)]),
}

# the entry points of the concordance-frame annotation and of each VCF-to-VCF tool, by name prefix, are bound on first use
# (load_annotation, load_low_af_ratio, ...), so that a build of the library without them, such as the host emulation of
# the filter path, still loads
_ANNOTATION, _AFR = ("ugvc_conc_annot",), ("ugvc_afr_", "ugvc_test_afr")
_BSN, _HCR = ("ugvc_bsn_", "ugvc_test_bsn"), ("ugvc_hcr_", "ugvc_test_hcr")
_BOUND_ON_USE = frozenset(n for n in SIGNATURES if n.startswith(_ANNOTATION + _AFR + _BSN + _HCR))
_groups_bound: set[tuple] = set()

_lib = None


def _bind(lib: C.CDLL, names):
    for name in names:
        res, args = SIGNATURES[name]
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args


def load_library() -> C.CDLL:
    """Load the shared library (once).  Raises if it was not built."""
    global _lib  # noqa: PLW0603
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                f"(make -C variantcalling_b200/csrc).  There is no CPU fallback for the hot path.")
        lib = C.CDLL(LIB_PATH)
        _bind(lib, [name for name in SIGNATURES if name not in _BOUND_ON_USE])
        _lib = lib
    return _lib


def _load_group(prefix: tuple) -> C.CDLL:
    """load_library() with the entry points named `prefix` bound.  Raises if the library lacks them."""
    lib = load_library()
    if prefix not in _groups_bound:
        _bind(lib, sorted(n for n in SIGNATURES if n.startswith(prefix)))
        _groups_bound.add(prefix)
    return lib


def load_annotation() -> C.CDLL:
    """load_library() with the annotation entry points bound.  Raises if the library lacks them."""
    return _load_group(_ANNOTATION)


def load_low_af_ratio() -> C.CDLL:
    """load_library() with the filter_low_af_ratio_to_background entry points bound.  Raises if the library lacks them."""
    return _load_group(_AFR)


def load_bridging_snvs() -> C.CDLL:
    """load_library() with the calibrate_bridging_snvs entry points bound.  Raises if the library lacks them."""
    return _load_group(_BSN)


def load_gvcf_hcr() -> C.CDLL:
    """load_library() with the gvcf_hcr entry points bound.  Raises if the library lacks them."""
    return _load_group(_HCR)


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    if isinstance(a, int):
        return C.c_void_p(a)
    raise TypeError(type(a))


class PinnedBuffer:
    """Page-locked host memory exposed as a numpy uint8 array."""

    def __init__(self, n_bytes: int):
        lib = load_library()
        p = C.c_void_p()
        rc = lib.ugvc_host_alloc(C.byref(p), max(1, n_bytes))
        if rc:
            raise UgvcError(rc, lib.ugvc_last_error(None).decode())
        self._p = p
        self.nbytes = n_bytes
        self.array = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(1, n_bytes),))

    @property
    def ptr(self) -> int:
        return self._p.value

    def free(self):
        if self._p:
            self.array = None
            load_library().ugvc_host_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.free()
        except Exception:  # noqa: BLE001, S110
            pass


def _file_edits(with_model: bool, recalibrate: bool, blacklists, end: np.ndarray | None):
    """A FileEdits struct and the arrays it points into (kept alive by the caller)."""
    bl = blacklists or []
    names = [a.encode() if isinstance(a, str) else bytes(a) for a, _ in bl]
    pos = [np.ascontiguousarray(p, dtype=np.int64) for _, p in bl]
    pos_all = np.concatenate(pos) if pos else np.zeros(0, np.int64)
    pos_off = np.concatenate(([0], np.cumsum([p.size for p in pos]))).astype(np.int64)
    name_buf = np.frombuffer(b"".join(names) or b"\0", dtype=np.uint8)
    name_off = np.concatenate(([0], np.cumsum([len(a) for a in names]))).astype(np.int64)
    e = FileEdits(int(bool(with_model)), int(bool(recalibrate)), len(bl), pos_all.ctypes.data if pos_all.size else None,
                  pos_off.ctypes.data, name_buf.ctypes.data, name_off.ctypes.data,
                  end.ctypes.data if end is not None else None, 0)
    return e, (pos_all, pos_off, name_buf, name_off)


class Context:
    """One GPU context (one per process/GPU)."""

    def __init__(self, device: int = 0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.ugvc_init(device, C.byref(h))
        if rc:
            raise UgvcError(rc, self.lib.ugvc_last_error(None).decode())
        self.h = h
        self.device = device
        self.n_features = self.n_classes = self.n_slots = 0
        self.cap_bytes = self.cap_records = 0

    def _check(self, rc: int):
        if rc == UGVC_OK:
            return
        msg = self.lib.ugvc_last_error(self.h).decode()
        if rc == UGVC_E_DATA:
            raise UgvcDataError(rc, msg)
        raise UgvcError(rc, msg)

    def _check_tool(self, rc: int, query, tool: str, lane: int):
        """_check for a VCF-to-VCF tool call: UGVC_E_DATA raises UgvcDataError with .<tool>_record / .<tool>_reason, the
        record the reference raises at and why, from the tool's error query (`query`, e.g. ugvc_afr_error)."""
        if rc == UGVC_E_DATA:
            rec, reason = C.c_int64(), C.c_int32()
            query(self.h, lane, C.byref(rec), C.byref(reason))
            err = UgvcDataError(rc, self.lib.ugvc_last_error(self.h).decode())
            setattr(err, f"{tool}_record", int(rec.value))
            setattr(err, f"{tool}_reason", int(reason.value))
            raise err
        self._check(rc)

    def close(self):
        if self.h:
            self.lib.ugvc_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001, S110
            pass

    # ---- setup
    def bind_thread(self):
        """Make this context's device current on the calling thread (before it allocates pinned memory)."""
        self._check(self.lib.ugvc_bind_thread(self.h))

    def load_plan(self, blob: bytes):
        buf = np.frombuffer(blob, dtype=np.uint8)
        self._check(self.lib.ugvc_load_plan(self.h, _ptr(buf), buf.size))
        f, k, s = C.c_int32(), C.c_int32(), C.c_int32()
        self._check(self.lib.ugvc_plan_info(self.h, C.byref(f), C.byref(k), C.byref(s)))
        self.n_features, self.n_classes, self.n_slots = f.value, k.value, s.value

    def set_key_order(self, info_keys: str | None, format_keys: str | None):
        """Tell K1 the usual INFO key order / FORMAT column (see :func:`learn_key_order`)."""
        self._check(self.lib.ugvc_set_key_order(self.h, (info_keys or "").encode(), (format_keys or "").encode()))

    def reserve(self, max_bytes: int, max_records: int, n_pipeline: int = 1):
        self._check(self.lib.ugvc_reserve(self.h, max_bytes, max_records, n_pipeline))
        self.cap_bytes, self.cap_records = max_bytes, (max_records + 127) // 128 * 128

    # ---- host-buffer hot path
    def alloc_outputs(self, n_max: int, want_recinfo: bool = True) -> dict:
        out = {"low_score": np.empty(n_max, np.uint8), "probs": np.empty((n_max, self.n_classes), np.float32),
               "qual": np.empty(n_max, np.float64)}
        if want_recinfo:
            out["recinfo"] = np.empty(n_max, RECINFO_DTYPE)
            out["line_start"] = np.empty(n_max + 1, np.int64)
        return out

    @staticmethod
    def trim_outputs(out: dict, n: int) -> dict:
        res = {k: (v[: n + 1] if k == "line_start" else v[:n]) for k, v in out.items()}
        res["n_records"] = n
        return res

    def filter_batch(self, text, threshold: float = 30.0, want_recinfo: bool = True) -> dict:
        """One batch of VCF data lines (bytes / uint8 array) -> dict of numpy results."""
        buf = np.frombuffer(text, dtype=np.uint8) if isinstance(text, (bytes, bytearray, memoryview)) else text
        n_max = max(1, int(np.count_nonzero(buf == 10)))  # noqa: PLR2004
        out = self.alloc_outputs(n_max, want_recinfo)
        n = C.c_int64()
        rc = self.lib.ugvc_filter_batch(self.h, _ptr(buf), buf.size, threshold, _ptr(out["low_score"]),
                                        _ptr(out["probs"]), _ptr(out["qual"]), _ptr(out.get("recinfo")),
                                        _ptr(out.get("line_start")), n_max, C.byref(n))
        self._check(rc)
        return self.trim_outputs(out, n.value)

    def submit(self, lane: int, text_ptr, n_bytes: int, threshold: float = 30.0):
        self._check(self.lib.ugvc_submit_batch(self.h, lane, _ptr(text_ptr), n_bytes, threshold))

    def submit_bgzf(self, lane: int, bgzf, n_bytes: int, threshold: float = 30.0):
        """Like :meth:`submit`, for whole BGZF blocks (compressed on the host, inflated on the device)."""
        self._check(self.lib.ugvc_submit_bgzf(self.h, lane, _ptr(bgzf), n_bytes, threshold))

    def inflate_bgzf(self, bgzf, want_text: bool = True) -> np.ndarray | int:
        """Inflate whole BGZF blocks on the device; returns the text (uint8 array) or just its size."""
        buf = np.frombuffer(bgzf, dtype=np.uint8) if isinstance(bgzf, (bytes, bytearray, memoryview)) else bgzf
        n = C.c_size_t()
        out = np.empty(self.cap_bytes, dtype=np.uint8) if want_text else None
        self._check(self.lib.ugvc_bgzf_inflate_device(self.h, _ptr(buf), buf.size, _ptr(out), 0 if out is None else out.size,
                                                      C.byref(n)))
        return out[: n.value] if want_text else int(n.value)

    def collect(self, lane: int, out: dict, capacity: int) -> int:
        n = C.c_int64()
        self._check(self.lib.ugvc_collect_batch(self.h, lane, _ptr(out.get("low_score")), _ptr(out.get("probs")),
                                                _ptr(out.get("qual")), _ptr(out.get("recinfo")),
                                                _ptr(out.get("line_start")), capacity, C.byref(n)))
        return n.value

    def predict_features(self, x: np.ndarray, threshold: float = 30.0) -> dict:
        """K3 on a dense (n, n_features) float32 matrix -> dict(low_score, probs, qual)."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        if x.ndim != 2 or x.shape[1] != self.n_features:
            raise ValueError(f"expected a (n, {self.n_features}) matrix, got {x.shape}")
        n = x.shape[0]
        out = self.alloc_outputs(max(1, n), want_recinfo=False)
        self._check(self.lib.ugvc_predict_features(self.h, _ptr(x) if n else None, n, x.shape[1], threshold,
                                                   _ptr(out["low_score"]), _ptr(out["probs"]), _ptr(out["qual"])))
        return self.trim_outputs(out, n)

    def enable_phreds(self, on: bool | int = True):
        """1/True: K3 keeps the per-class phreds; 2: the fp64 class likelihoods (--treat_multiallelics)."""
        self._check(self.lib.ugvc_enable_phreds(self.h, int(on)))

    def collect_phreds(self, lane: int, n: int) -> np.ndarray:
        out = np.empty((max(1, n), self.n_classes), np.float64)
        self._check(self.lib.ugvc_collect_phreds(self.h, lane, _ptr(out), out.shape[0]))
        return out[:n]

    # ---- device-resident hot path (pointers are ints, e.g. torch.Tensor.data_ptr())
    def filter_device(self, d_text: int, n_bytes: int, threshold: float, d_low: int, d_probs: int, d_qual: int,
                      capacity: int, d_n_records: int = 0, stream: int = 0, d_recinfo: int = 0,
                      d_line_start: int = 0, lane: int = 0):
        self._check(self.lib.ugvc_filter_device_lane(self.h, lane, d_text, n_bytes, threshold, d_low, d_probs, d_qual,
                                                     d_recinfo or None, d_line_start or None, capacity,
                                                     d_n_records or None, stream or None))

    def device_status(self, stream: int = 0, lane: int = 0):
        self._check(self.lib.ugvc_device_status_lane(self.h, lane, stream or None))

    # ---- file to file on the device
    def filter_bgzf(self, bgzf: np.ndarray, skip_head: int, take_bytes: int, threshold: float, flags: int, max_records: int,
                    lane: int = 0, bufs: dict | None = None) -> dict | None:
        """One range of whole lines: compressed blocks in, filtered + scored + edited records out as BGZF blocks
        (see ugvc_filter_bgzf).  Returns None when the range needs the general host writer."""
        return self._filter_bgzf(bgzf, skip_head, take_bytes, threshold, flags, max_records, lane, bufs, None)

    def filter_bgzf_edits(self, bgzf: np.ndarray, skip_head: int, take_bytes: int, threshold: float, flags: int,
                          max_records: int, *, with_model: bool = True, recalibrate_genotype: bool = False,
                          blacklists: list[tuple[str, np.ndarray]] | None = None, want_end: bool = False, lane: int = 0,
                          bufs: dict | None = None) -> dict | None:
        """:meth:`filter_bgzf` with the rest of the record edits (see ugvc_filter_bgzf_edits): a model-less plan
        (with_model=False), --recalibrate_genotype (needs enable_phreds(1) before reserve), blacklists as
        [(annotation, sorted POS of the range's contig)], and with want_end the INFO/END of every record ("end", 0 where
        there is none).  The result also holds "n_blacklisted".  None when the range needs the general host writer."""
        end = None
        if want_end:
            end = bufs["end"] if bufs is not None and "end" in bufs else np.empty(max(1, max_records), np.int64)
        e, keep = _file_edits(with_model, recalibrate_genotype, blacklists, end)
        res = self._filter_bgzf(bgzf, skip_head, take_bytes, threshold, flags, max_records, lane, bufs, e)
        if res is not None:
            res["n_blacklisted"] = int(e.n_blacklisted)
            if end is not None:
                res["end"] = end[: res["n_records"]]
        return res

    def filter_bgzf_split(self, bgzf: np.ndarray, skip_head: int, take_bytes: int, threshold: float, flags: int,
                          max_records: int, *, index_ctx: "Context", ma, ref: np.ndarray, split_stats: np.ndarray,
                          recalibrate_genotype: bool = False, blacklists: list[tuple[str, np.ndarray]] | None = None,
                          want_end: bool = False, lane: int = 0, bufs: dict | None = None) -> dict | None:
        """--treat_multiallelics on the file path (see ugvc_filter_bgzf_split): one whole contig, with `index_ctx` (the
        model-less plan, reserved with this lane) for the index pass, `ma` (a ugvc_ma handle) for the split and `ref` (the
        contig's sequence, uint8) -- results as :meth:`filter_bgzf_edits`.  Needs enable_phreds(2) before reserve.
        `split_stats` (int64[8]) receives out_split; the reference's failures come back as UgvcDataError (see
        multiallelics.DeviceSplitPlan.filter_bgzf, which maps them).  None when the contig needs the host path."""
        end = None
        if want_end:
            end = bufs["end"] if bufs is not None and "end" in bufs else np.empty(max(1, max_records), np.int64)
        e, keep = _file_edits(True, recalibrate_genotype, blacklists, end)  # noqa: F841  (keep: alive for the call)
        ref = np.ascontiguousarray(ref, dtype=np.uint8)
        res = self._filter_bgzf(bgzf, skip_head, take_bytes, threshold, flags, max_records, lane, bufs, e,
                                split=(index_ctx.h, ma, ref, split_stats))
        if res is not None:
            res["n_blacklisted"] = int(e.n_blacklisted)
            if end is not None:
                res["end"] = end[: res["n_records"]]
        return res

    def filter_bgzf_split_stage_ms(self, lane: int = 0) -> list[float]:
        """ms of the last filter_bgzf_split call on `lane`: H2D + inflate, index K1, split build, scored K1..K3,
        merge + score, record writer, deflate + pack, D2H."""
        ms = (C.c_float * 8)()
        self._check(self.lib.ugvc_filter_bgzf_split_stage_ms(self.h, lane, C.cast(ms, C.c_void_p)))
        return list(ms)

    def test_ma_score(self, lik: np.ndarray, threshold: float) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The split path's score kernel on (n, width) likelihoods (test hook ugvc_test_ma_score): phreds, qual, low."""
        lik = np.ascontiguousarray(lik, dtype=np.float64)
        n, width = lik.shape
        ph, q, low = np.empty_like(lik), np.empty(n, np.float64), np.empty(n, np.uint8)
        self._check(self.lib.ugvc_test_ma_score(self.h, _ptr(lik), n, width, threshold, _ptr(ph), _ptr(q), _ptr(low)))
        return ph, q, low

    def test_write_records(self, text, line_start, recinfo, flags: int, *, low_score=None, qual=None, phreds=None,
                           with_model: bool = True, recalibrate_genotype: bool = False, blacklists=None,
                           want_end: bool = False) -> dict | None:
        """The device record writer alone on caller records (ugvc_test_write_records): {"text", "line_start",
        "n_blacklisted"[, "end"]}, or None when it hands the records back."""
        buf = np.frombuffer(text, dtype=np.uint8) if isinstance(text, (bytes, bytearray)) else np.ascontiguousarray(text)
        ls = np.ascontiguousarray(line_start, dtype=np.int64)
        ri = np.ascontiguousarray(recinfo)
        n = ls.size - 1
        end = np.zeros(max(1, n), np.int64) if want_end else None
        e, keep = _file_edits(with_model, recalibrate_genotype, blacklists, end)  # noqa: F841  (keep: alive for the call)
        ph = None if phreds is None else np.ascontiguousarray(phreds, dtype=np.float64)
        low = None if low_score is None else np.ascontiguousarray(low_score, dtype=np.uint8)
        q = None if qual is None else np.ascontiguousarray(qual, dtype=np.float64)
        out = np.empty(buf.size + n * 256 + 4096, dtype=np.uint8)
        out_ls = np.empty(n + 1, dtype=np.int64)
        nb = self.lib.ugvc_test_write_records(self.h, _ptr(buf), buf.size, _ptr(ls), _ptr(ri), n, _ptr(low), _ptr(q), _ptr(ph),
                                              0 if ph is None else (ph.shape[1] if ph.ndim == 2 else 0), flags, C.byref(e),
                                              _ptr(out), out.size, _ptr(out_ls))
        if nb == UGVC_E_FALLBACK:
            return None
        if nb < 0:
            self._check(int(nb))
        res = {"text": out[:nb].tobytes(), "line_start": out_ls, "n_blacklisted": int(e.n_blacklisted)}
        if end is not None:
            res["end"] = end[:n]
        return res

    def _filter_bgzf(self, bgzf, skip_head, take_bytes, threshold, flags, max_records, lane, bufs, edits, split=None):
        comp = np.ascontiguousarray(bgzf, dtype=np.uint8)
        if bufs is not None:  # the caller's (pinned, reused) buffers: out, blocks, ri, ls, low
            out, blocks, ri, ls, low = bufs["out"], bufs["blocks"], bufs["ri"], bufs["ls"], bufs["low"]
        else:
            n_text_max = (take_bytes or comp.size * 64) + max_records * 64 + 65536
            out = np.empty(n_text_max // DEF_CHUNK * 65536 + 65536 if take_bytes else comp.size * 8 + (1 << 20), dtype=np.uint8)
            blocks = np.empty(out.size // 65536 + 8, dtype=np.uint32)
            ri = np.empty(max_records, dtype=RECINFO_DTYPE)
            ls = np.empty(max_records + 1, dtype=np.int64)
            low = np.empty(max_records, dtype=np.uint8)
        nb, nblk, n = C.c_size_t(), C.c_size_t(), C.c_int64()
        args = (_ptr(out), out.size, C.byref(nb), _ptr(blocks), blocks.size, C.byref(nblk), _ptr(ri), _ptr(ls), _ptr(low),
                max_records, C.byref(n))
        if split is not None:
            idx_h, ma, ref, stats = split
            rc = self.lib.ugvc_filter_bgzf_split(self.h, idx_h, ma, lane, _ptr(comp), comp.size, skip_head, take_bytes,
                                                 _ptr(ref) if ref.size else None, ref.size, threshold, flags, C.byref(edits),
                                                 *args, _ptr(stats))
        elif edits is None:
            rc = self.lib.ugvc_filter_bgzf(self.h, lane, _ptr(comp), comp.size, skip_head, take_bytes, threshold, flags, *args)
        else:
            rc = self.lib.ugvc_filter_bgzf_edits(self.h, lane, _ptr(comp), comp.size, skip_head, take_bytes, threshold, flags,
                                                 C.byref(edits), *args)
        if rc == UGVC_E_FALLBACK:
            return None
        self._check(rc)
        k = n.value
        return {"n_records": k, "bgzf": out[: nb.value], "block_csize": blocks[: nblk.value], "recinfo": ri[:k],
                "line_start": ls[: k + 1], "low_score": low[:k]}

    def afr_bgzf(self, data: np.ndarray, skip_head: int, take_bytes: int, is_text: bool, params: AfrParams, max_records: int,
                 lane: int = 0) -> dict:
        """filter_low_af_ratio_to_background on one range of whole lines (ugvc_afr_bgzf): BGZF blocks (or, with is_text,
        the plain text) in, BGZF blocks of the edited records out.  Needs the model-less plan and reserve() sized for the
        range.  A record the reference raises at comes back as UgvcDataError with .afr_record / .afr_reason set."""
        lib = load_low_af_ratio()
        src = np.ascontiguousarray(data, dtype=np.uint8)
        n_text = take_bytes or (src.size if is_text else src.size * 64)
        out = np.empty(n_text // DEF_CHUNK * 65536 + n_text // 8 + max_records * (AFR_MAX_FILTER_BYTES + 1) + (1 << 20), np.uint8)
        blocks = np.empty(out.size // 65536 + 8, dtype=np.uint32)
        ri = np.empty(max(1, max_records), dtype=RECINFO_DTYPE)
        ls = np.empty(max_records + 1, dtype=np.int64)
        end = np.empty(max(1, max_records), dtype=np.int64)
        flags = np.empty(max(1, max_records), dtype=np.uint8)
        nb, nblk, n, nf = C.c_size_t(), C.c_size_t(), C.c_int64(), C.c_int64()
        rc = lib.ugvc_afr_bgzf(self.h, lane, _ptr(src), src.size, skip_head, take_bytes, int(bool(is_text)), C.byref(params),
                               _ptr(out), out.size, C.byref(nb), _ptr(blocks), blocks.size, C.byref(nblk), _ptr(ri), _ptr(ls),
                               _ptr(end), _ptr(flags), max_records, C.byref(n), C.byref(nf))
        self._check_tool(rc, lib.ugvc_afr_error, "afr", lane)
        k = n.value
        return {"n_records": k, "n_filtered": int(nf.value), "bgzf": out[: nb.value], "block_csize": blocks[: nblk.value],
                "recinfo": ri[:k], "line_start": ls[: k + 1], "end": end[:k], "flags": flags[:k]}

    def afr_stage_ms(self, lane: int = 0) -> list[float]:
        """ms of the last afr_bgzf call on `lane`: H2D + inflate, index K1, decide + scan + copy, deflate + pack, D2H."""
        ms = (C.c_float * 5)()
        self._check(load_low_af_ratio().ugvc_afr_stage_ms(self.h, lane, C.cast(ms, C.c_void_p)))
        return list(ms)

    def bsn_add_contig(self, name: str, seq: bytes):
        """Upload one FASTA contig (raw bytes) to the context's calibrate_bridging_snvs contig table."""
        buf = np.frombuffer(seq, dtype=np.uint8)
        self._check(load_bridging_snvs().ugvc_bsn_add_contig(self.h, name.encode(), _ptr(buf) if buf.size else None, buf.size))

    def bsn_clear_contigs(self):
        self._check(load_bridging_snvs().ugvc_bsn_clear_contigs(self.h))

    def bsn_bgzf(self, data: np.ndarray, skip_head: int, take_bytes: int, is_text: bool, params: BsnParams, max_records: int,
                 lane: int = 0) -> dict:
        """calibrate_bridging_snvs on one range of whole lines (ugvc_bsn_bgzf), in the shape of afr_bgzf, plus "hmer" and
        "src_line_start" (line starts in the range's input text).  A record the reference raises at comes back as
        UgvcDataError with .bsn_record / .bsn_reason set."""
        lib = load_bridging_snvs()
        src = np.ascontiguousarray(data, dtype=np.uint8)
        n_text = take_bytes or (src.size if is_text else src.size * 64)
        out = np.empty(n_text // DEF_CHUNK * 65536 + n_text // 8 + max_records * (BSN_MAX_QUAL_BYTES + 5) + (1 << 20), np.uint8)
        blocks = np.empty(out.size // 65536 + 8, dtype=np.uint32)
        ri = np.empty(max(1, max_records), dtype=RECINFO_DTYPE)
        ls = np.empty(max_records + 1, dtype=np.int64)
        src_ls = np.empty(max_records + 1, dtype=np.int64)
        end = np.empty(max(1, max_records), dtype=np.int64)
        flags = np.empty(max(1, max_records), dtype=np.uint8)
        hmer = np.empty(max(1, max_records), dtype=np.int32)
        nb, nblk, n, nr = C.c_size_t(), C.c_size_t(), C.c_int64(), C.c_int64()
        rc = lib.ugvc_bsn_bgzf(self.h, lane, _ptr(src), src.size, skip_head, take_bytes, int(bool(is_text)), C.byref(params),
                               _ptr(out), out.size, C.byref(nb), _ptr(blocks), blocks.size, C.byref(nblk), _ptr(ri), _ptr(ls),
                               _ptr(src_ls), _ptr(end), _ptr(flags), _ptr(hmer), max_records, C.byref(n), C.byref(nr))
        self._check_tool(rc, lib.ugvc_bsn_error, "bsn", lane)
        k = n.value
        return {"n_records": k, "n_rescued": int(nr.value), "bgzf": out[: nb.value], "block_csize": blocks[: nblk.value],
                "recinfo": ri[:k], "line_start": ls[: k + 1], "src_line_start": src_ls[: k + 1], "end": end[:k],
                "flags": flags[:k], "hmer": hmer[:k]}

    def bsn_stage_ms(self, lane: int = 0) -> list[float]:
        """ms of the last bsn_bgzf call on `lane`: H2D + inflate, index K1, decide + scan + copy, deflate + pack, D2H."""
        ms = (C.c_float * 5)()
        self._check(load_bridging_snvs().ugvc_bsn_stage_ms(self.h, lane, C.cast(ms, C.c_void_p)))
        return list(ms)

    def hcr_scan(self, data: np.ndarray, skip_head: int, take_bytes: int, params: HcrParams, max_records: int,
                 lane: int = 0) -> dict:
        """The first half of gvcf_hcr on one range of whole lines of BGZF blocks (ugvc_hcr_scan): inflate, index, decide
        and the per-contig prefix max; the piece stays on the lane for hcr_emit.  {"n_records", "runs" ((record, line
        start) of each record that starts a contig run, by record), "r0", "first_start", "last_start"}."""
        lib = load_gvcf_hcr()
        src = np.ascontiguousarray(data, dtype=np.uint8)
        runs = np.empty((max(1, max_records), 2), dtype=np.int64)
        stats = np.zeros(4, dtype=np.int64)
        n = C.c_int64()
        self._check(lib.ugvc_hcr_scan(self.h, lane, _ptr(src), src.size, skip_head, take_bytes, C.byref(params), max_records,
                                      C.byref(n), _ptr(stats), _ptr(runs)))
        runs = runs[: int(stats[0])]
        return {"n_records": n.value, "runs": runs[np.argsort(runs[:, 0])], "r0": int(stats[1]),
                "first_start": int(stats[2]), "last_start": int(stats[3])}

    def hcr_emit(self, params: HcrParams, continues_contig: bool, entry_extent: int, capacity: int, lane: int = 0) -> dict:
        """The second half (ugvc_hcr_emit) on the piece `lane` holds: {"bed" (bytes), "n_lines", "skipped",
        "exit_extent", "longest_segment"}.  A record the reference raises at comes back as UgvcDataError with
        .hcr_record / .hcr_reason set."""
        lib = load_gvcf_hcr()
        out = np.empty(max(1, capacity), dtype=np.uint8)
        stats = np.zeros(4, dtype=np.int64)
        nb = C.c_size_t()
        rc = lib.ugvc_hcr_emit(self.h, lane, C.byref(params), int(bool(continues_contig)), int(entry_extent), _ptr(out), out.size,
                               C.byref(nb), _ptr(stats))
        self._check_tool(rc, lib.ugvc_hcr_error, "hcr", lane)
        return {"bed": out[: nb.value].tobytes(), "n_lines": int(stats[0]), "skipped": int(stats[1]),
                "exit_extent": int(stats[2]), "longest_segment": int(stats[3])}

    def hcr_stage_ms(self, lane: int = 0) -> list[float]:
        """ms of the last scan + emit on `lane`: H2D + inflate, index K1, decide + prefix max, emit kernels, D2H."""
        ms = (C.c_float * 5)()
        self._check(load_gvcf_hcr().ugvc_hcr_stage_ms(self.h, lane, C.cast(ms, C.c_void_p)))
        return list(ms)

    def filter_bgzf_first_records(self, text_offsets, lane: int = 0) -> np.ndarray:
        """Index of the first record at or after each byte offset of the last filter_bgzf range's text."""
        off = np.ascontiguousarray(text_offsets, dtype=np.uint64)
        out = np.empty(off.size, dtype=np.int64)
        self._check(self.lib.ugvc_filter_bgzf_first_records(self.h, lane, _ptr(off), off.size, _ptr(out)))
        return out

    def filter_bgzf_stage_ms(self, lane: int = 0) -> list[float]:
        ms = (C.c_float * 5)()
        self._check(self.lib.ugvc_filter_bgzf_stage_ms(self.h, lane, C.cast(ms, C.c_void_p)))
        return list(ms)

    # ---- the one collective of the path, through the C ABI (NCCL bound at run time)
    @staticmethod
    def nccl_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        rc = load_library().ugvc_nccl_unique_id(C.cast(buf, C.c_void_p))
        if rc:
            raise UgvcError(rc, load_library().ugvc_last_error(None).decode())
        return bytes(buf)

    def nccl_comm_init(self, unique_id: bytes, world_size: int, rank: int) -> int:
        comm = C.c_void_p()
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(self.lib.ugvc_nccl_comm_init(self.h, C.cast(buf, C.c_void_p), world_size, rank, C.byref(comm)))
        return comm.value

    def nccl_comm_destroy(self, comm: int):
        self.lib.ugvc_nccl_comm_destroy(comm)

    def counts_allreduce(self, comm: int, stream: int = 0) -> dict:
        """Sum the pass / fail counter block over the ranks of `comm` (ncclAllReduce, in place) and read it."""
        out = (C.c_int64 * 4)()
        self._check(self.lib.ugvc_counts_allreduce(self.h, comm, C.cast(out, C.c_void_p), stream or None))
        return {"n_records": out[0], "n_low_score": out[1], "n_pass": out[2], "n_cg": out[3]}

    def synth_device(self, seed: int, first: int, n: int, total: int, n_custom: int, d_text: int, capacity: int,
                     stream: int = 0) -> int:
        nb = C.c_size_t()
        self._check(self.lib.ugvc_synth_device(self.h, seed, first, n, total, n_custom, d_text, capacity,
                                               C.byref(nb), stream or None))
        return nb.value

    # ---- counters / introspection
    def counts_reset(self):
        self._check(self.lib.ugvc_counts_reset(self.h))

    def counts(self) -> dict:
        c = Counts()
        self._check(self.lib.ugvc_counts_get(self.h, C.byref(c)))
        return {"n_records": c.n_records, "n_low_score": c.n_low_score, "n_pass": c.n_pass, "n_cg": c.n_cg}

    def counts_device_ptr(self) -> int:
        p = C.c_void_p()
        self._check(self.lib.ugvc_counts_device_ptr(self.h, C.byref(p)))
        return p.value

    def debug_features(self, n: int, lane: int = 0) -> np.ndarray:
        out = np.empty((self.n_features, max(1, n)), np.float32)
        self._check(self.lib.ugvc_debug_features(self.h, lane, _ptr(out), out.size))
        return out[:, :n]

    def debug_raw(self, n: int, lane: int = 0) -> np.ndarray:
        out = np.empty((self.n_slots, max(1, n)), np.uint32)
        self._check(self.lib.ugvc_debug_raw(self.h, lane, _ptr(out), out.size))
        return out[:, :n]

    def slow_records(self, lane: int = 0) -> int:
        """Records of the lane's last batch that went through the generic parser (diagnostic)."""
        return int(self.lib.ugvc_debug_slow_records(self.h, lane))

    def last_data_error(self) -> tuple[int, int, int]:
        r, c, k = C.c_int64(), C.c_int32(), C.c_int32()
        self.lib.ugvc_last_data_error(self.h, C.byref(r), C.byref(c), C.byref(k))
        return r.value, c.value, k.value

    def launch_count(self) -> int:
        return int(self.lib.ugvc_launch_count(self.h))

    def k3_config(self) -> dict:
        """The K3 launch the loaded plan gets (test hook ugvc_test_k3_config)."""
        out = np.zeros(10, np.int32)
        self._check(self.lib.ugvc_test_k3_config(self.h, _ptr(out)))
        kernel, tpb, nbuf, groups, nch, chunk, resident, grid, walk, split = (int(v) for v in out)
        return {"kernel": ("heap", "infer")[kernel], "tpb": tpb, "nbuf": nbuf, "groups": groups, "nch": nch, "chunk": chunk,
                "resident": bool(resident), "grid": grid, "gs": tpb // groups // split, "split": split,
                "walk": ("plain", "categorical")[walk]}

    def test_format_g(self, values) -> np.ndarray:
        """The record writer's "%g" on the device (test hook ugvc_test_format_g): an (n, 16) uint8 array, text in
        bytes 0..14, its length in byte 15 (0 = left to the host writer)."""
        v = np.ascontiguousarray(values, dtype=np.float32)
        out = np.empty((v.size, 16), np.uint8)
        if v.size:
            self._check(self.lib.ugvc_test_format_g(self.h, _ptr(v), v.size, _ptr(out)))
        return out

    def test_device_deflate(self, data: bytes, encoder: int = 0) -> tuple[bytes, np.ndarray]:
        """The file path's BGZF encoder on `data` (test hook ugvc_test_device_deflate; 0 = warp per block, 1 = thread
        per block): (packed blocks, compressed size of each block).  Needs reserve() sized for the bytes."""
        buf = np.frombuffer(data, dtype=np.uint8)
        n_blocks = (buf.size + DEF_CHUNK - 1) // DEF_CHUNK
        out = np.empty(n_blocks * 65536 + 1, np.uint8)
        csize = np.empty(n_blocks + 1, np.uint32)
        nb, nblk = C.c_size_t(), C.c_size_t()
        self._check(self.lib.ugvc_test_device_deflate(self.h, _ptr(buf) if buf.size else None, buf.size, encoder, _ptr(out),
                                                      out.size, _ptr(csize), csize.size, C.byref(nb), C.byref(nblk)))
        return out[: nb.value].tobytes(), csize[: nblk.value].copy()

    def test_device_inflate(self, bgzf: bytes, decoder: int = 0) -> tuple[np.ndarray, np.ndarray]:
        """The device BGZF decoder on whole BGZF blocks (test hook ugvc_test_device_inflate; 0 = warp per block, 1 =
        thread per block): (inflated bytes, INF_* code of each block with ISIZE > 0).  Needs reserve() sized for the
        output; a failed block's bytes are unspecified."""
        buf = np.frombuffer(bgzf, dtype=np.uint8)
        out = np.empty(max(1, self.cap_bytes), np.uint8)
        rc = np.empty(max(1, buf.size // 26 + 1), np.int32)  # a BGZF block is at least 26 bytes
        n, nblk = C.c_size_t(), C.c_size_t()
        self._check(self.lib.ugvc_test_device_inflate(self.h, _ptr(buf) if buf.size else None, buf.size, decoder, _ptr(out),
                                                      out.size, C.byref(n), _ptr(rc), rc.size, C.byref(nblk)))
        return out[: n.value], rc[: nblk.value].copy()

    def enable_stage_timing(self, on: bool = True):
        self._check(self.lib.ugvc_enable_stage_timing(self.h, int(on)))

    def stage_ms(self) -> tuple[list[float], int]:
        """(summed ms of K0..K3, number of enqueues) since stage timing was enabled."""
        arr = (C.c_float * 4)()
        n = C.c_int64()
        self._check(self.lib.ugvc_stage_ms(self.h, arr, C.byref(n)))
        return list(arr), n.value


def _lines(text: bytes) -> tuple[np.ndarray, np.ndarray, int]:
    """(bytes, line starts with the end after them, line count) of whole lines, for the kernel test hooks."""
    buf = np.frombuffer(text, dtype=np.uint8)
    ls = np.concatenate(([0], np.flatnonzero(buf == 10) + 1)).astype(np.int64)  # noqa: PLR2004
    return buf, ls, ls.size - 1


def test_afr(text: bytes, params: AfrParams) -> dict:
    """The filter_low_af_ratio_to_background kernels alone on whole lines (test hook ugvc_test_afr, no context):
    {"text", "line_start", "failed", "end", "n_filtered"}, or {"error": (record, reason)} where the reference raises."""
    lib = load_low_af_ratio()
    buf, ls, n = _lines(text)
    out = np.empty(buf.size + n * (AFR_MAX_FILTER_BYTES + 1) + 16, np.uint8)
    out_ls = np.empty(n + 1, np.int64)
    failed = np.empty(max(1, n), np.uint8)
    end = np.empty(max(1, n), np.int64)
    nf, rec, reason = C.c_int64(), C.c_int64(), C.c_int32()
    nb = lib.ugvc_test_afr(_ptr(buf) if buf.size else None, buf.size, _ptr(ls), n, C.byref(params), _ptr(out), out.size,
                           _ptr(out_ls), _ptr(failed), _ptr(end), C.byref(nf), C.byref(rec), C.byref(reason))
    if nb == UGVC_E_DATA:
        return {"error": (int(rec.value), int(reason.value))}
    if nb < 0:
        raise UgvcError(int(nb), "ugvc_test_afr failed")
    return {"text": out[:nb].tobytes(), "line_start": out_ls, "failed": failed[:n].astype(bool), "end": end[:n],
            "n_filtered": int(nf.value)}


def test_bsn(text: bytes, contigs: dict, params: BsnParams) -> dict:
    """The calibrate_bridging_snvs kernels alone on whole lines and the given contigs ({name: bytes}; test hook
    ugvc_test_bsn, no context): {"text", "line_start", "rescued", "hmer", "end", "n_rescued"}, or {"error": (record,
    reason)} where the reference raises."""
    lib = load_bridging_snvs()
    buf, ls, n = _lines(text)
    names = [k.encode() for k in contigs]
    name_buf = np.frombuffer(b"".join(names) or b"\0", dtype=np.uint8)
    name_off = np.concatenate(([0], np.cumsum([len(k) for k in names]))).astype(np.int64)
    seq_buf = np.frombuffer(b"".join(contigs.values()) or b"\0", dtype=np.uint8)
    seq_off = np.concatenate(([0], np.cumsum([len(v) for v in contigs.values()]))).astype(np.int64)
    out = np.empty(buf.size + n * (BSN_MAX_QUAL_BYTES + 5) + 16, np.uint8)
    out_ls = np.empty(n + 1, np.int64)
    rescued = np.empty(max(1, n), np.uint8)
    hmer = np.empty(max(1, n), np.int32)
    end = np.empty(max(1, n), np.int64)
    nr, rec, reason = C.c_int64(), C.c_int64(), C.c_int32()
    nb = lib.ugvc_test_bsn(_ptr(buf) if buf.size else None, buf.size, _ptr(ls), n, _ptr(name_buf), _ptr(name_off), _ptr(seq_buf),
                           _ptr(seq_off), len(names), C.byref(params), _ptr(out), out.size, _ptr(out_ls), _ptr(rescued),
                           _ptr(hmer), _ptr(end), C.byref(nr), C.byref(rec), C.byref(reason))
    if nb == UGVC_E_DATA:
        return {"error": (int(rec.value), int(reason.value))}
    if nb < 0:
        raise UgvcError(int(nb), "ugvc_test_bsn failed")
    return {"text": out[:nb].tobytes(), "line_start": out_ls, "rescued": rescued[:n].astype(bool), "hmer": hmer[:n],
            "end": end[:n], "n_rescued": int(nr.value)}


def test_hcr(text: bytes, params: HcrParams, continues_contig: bool = False, entry_extent: int = -1, seg_bound: int = 0) -> dict:
    """The gvcf_hcr kernels alone on whole lines with the given entry state (test hook ugvc_test_hcr, no context):
    {"bed", "flags", "n_lines", "skipped", "exit_extent", "longest_segment"}, or {"error": (record, reason)} where the
    reference raises."""
    lib = load_gvcf_hcr()
    buf, ls, n = _lines(text)
    out = np.empty(buf.size + 48 * n + 16, np.uint8)
    flags = np.empty(max(1, n), np.uint8)
    stats = np.zeros(4, np.int64)
    rec, reason = C.c_int64(), C.c_int32()
    nb = lib.ugvc_test_hcr(_ptr(buf) if buf.size else None, buf.size, _ptr(ls), n, C.byref(params), int(bool(continues_contig)),
                           int(entry_extent), int(seg_bound), _ptr(out), out.size, _ptr(flags), _ptr(stats), C.byref(rec),
                           C.byref(reason))
    if nb == UGVC_E_DATA:
        return {"error": (int(rec.value), int(reason.value))}
    if nb < 0:
        raise UgvcError(int(nb), "ugvc_test_hcr failed")
    return {"bed": out[:nb].tobytes(), "flags": flags[:n].copy(), "n_lines": int(stats[0]), "skipped": int(stats[1]),
            "exit_extent": int(stats[2]), "longest_segment": int(stats[3])}


def synth_header(n_custom: int) -> str:
    lib = load_library()
    n = lib.ugvc_synth_header(n_custom, None, 0)
    buf = C.create_string_buffer(int(n))
    lib.ugvc_synth_header(n_custom, buf, n)
    return buf.raw.decode()


def learn_key_order(sample: bytes, max_records: int = 2000, min_presence: float = 0.0) -> tuple[str, str]:
    """Order of the INFO keys and the most common FORMAT column over the first records of
    ``sample`` (VCF data lines).

    Every record contributes the chain key[i] -> key[i+1]; a topological order of the union
    graph is a common supersequence of all the records' key sequences (records written by
    GATK/htsjdk carry their keys sorted, optional keys simply missing).  Keys caught in a cycle
    (files mixing orders) are left out and take K1's generic lookup path, and so can keys present
    in fewer than ``min_presence`` of the records (default 0: even the 15 %-present annotations of the cfg-3
    input are scheduled rather than left to the generic path)."""
    import heapq

    first_seen: dict[str, int] = {}
    seen_in: dict[str, int] = {}
    succ: dict[str, set] = {}
    indeg: dict[str, int] = {}
    formats: dict[str, int] = {}
    n = 0
    for line in sample.split(b"\n"):
        if not line or line.startswith(b"#"):
            continue
        cols = line.split(b"\t")
        if len(cols) < 8:  # noqa: PLR2004
            continue
        n += 1
        if n > max_records:
            break
        if len(cols) > 8:  # noqa: PLR2004
            f = cols[8].decode("latin-1")
            formats[f] = formats.get(f, 0) + 1
        if cols[7] == b".":
            continue
        prev = None
        for kv in cols[7].split(b";"):
            if not kv:
                continue
            key, sep, _ = kv.partition(b"=")
            name = key.decode("latin-1") + ("" if sep else "!")
            if ";" in name or len(name) > 24:  # noqa: PLR2004
                prev = None
                continue
            if name not in first_seen:
                first_seen[name] = len(first_seen)
                succ[name] = set()
                indeg[name] = 0
            seen_in[name] = seen_in.get(name, 0) + 1
            if prev is not None and prev != name and name not in succ[prev]:
                succ[prev].add(name)
                indeg[name] += 1
            prev = name
    heap = [(first_seen[k], k) for k, d in indeg.items() if d == 0]
    heapq.heapify(heap)
    order = []
    while heap:
        _, k = heapq.heappop(heap)
        order.append(k)
        for m in succ[k]:
            indeg[m] -= 1
            if indeg[m] == 0:
                heapq.heappush(heap, (first_seen[m], m))
    n_seen = max(1, min(n, max_records))
    order = [k for k in order if seen_in.get(k, 0) >= min_presence * n_seen]
    fmt = max(formats, key=formats.get) if formats else ""
    return ";".join(order[:128]), fmt if len(fmt) <= 24 else ""  # noqa: PLR2004
