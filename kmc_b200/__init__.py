"""kmc_b200 — Python host side over the C ABI (include/kmc_b200.h) of the H100 stage-2 path of KMC.

The product is the CUDA library `libkmc_b200.so` (kmc_b200/csrc); this module is a thin ctypes mirror used
by the tests and by bench.py.  Names follow the reference: a *bin* of super-k-mers goes through
Expand -> Sort -> Compact exactly like `CKmerBinSorter<SIZE>::ProcessBins` (kmc_core/kb_sorter.h:210-237).
There is no CPU fallback: constructing a `Stage2Context` without an H100 raises.
"""
import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.abspath(os.environ["KMCB200_LIB"]) if os.environ.get("KMCB200_LIB") else os.path.join(_HERE, "libkmc_b200.so")      # KMCB200_LIB: experiment builds (kmc_b200.build.build_variant)

OK, ERR_INVALID, ERR_NO_DEVICE, ERR_CUDA, ERR_BIN_FORMAT, ERR_CAPACITY, ERR_BUSY = 0, -1, -2, -3, -4, -5, -6


class KmcB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("kmc_b200 error %d: %s" % (code, msg))
        self.code = code


class _Params(C.Structure):
    _fields_ = [("kmer_len", C.c_uint32), ("both_strands", C.c_uint32), ("cutoff_min", C.c_uint32), ("cutoff_max", C.c_uint32),
                ("counter_max", C.c_uint32), ("lut_prefix_len", C.c_uint32), ("device", C.c_int32), ("n_slots", C.c_uint32)]


class _DbParams(C.Structure):
    _fields_ = [("kmer_len", C.c_uint32), ("counter_size", C.c_uint32), ("lut_prefix_len", C.c_uint32), ("signature_len", C.c_uint32),
                ("cutoff_min", C.c_uint32), ("cutoff_max", C.c_uint32), ("both_strands", C.c_uint32)]


class _SplitParams(C.Structure):
    _fields_ = [("kmer_len", C.c_uint32), ("signature_len", C.c_uint32), ("n_bins", C.c_uint32), ("device", C.c_int32), ("max_batch_bytes", C.c_uint64)]


class _SigstatsParams(C.Structure):
    _fields_ = [("kmer_len", C.c_uint32), ("signature_len", C.c_uint32), ("device", C.c_int32), ("reserved", C.c_uint32), ("max_batch_bytes", C.c_uint64)]


class _SmallKParams(C.Structure):
    _fields_ = [("kmer_len", C.c_uint32), ("both_strands", C.c_uint32), ("device", C.c_int32), ("reserved", C.c_uint32), ("max_batch_bytes", C.c_uint64)]


class _EstimatorParams(C.Structure):
    _fields_ = [("kmer_len", C.c_uint32), ("s", C.c_uint32), ("device", C.c_int32), ("reserved", C.c_uint32), ("max_batch_bytes", C.c_uint64)]


class _FastxParams(C.Structure):
    _fields_ = [("device", C.c_int32), ("format", C.c_uint32), ("max_chunk_bytes", C.c_uint64)]


class _KmcDbParams(C.Structure):
    _fields_ = [("device", C.c_int32), ("kmer_len", C.c_uint32), ("lut_prefix_len", C.c_uint32), ("counter_size", C.c_uint32),
                ("min_count", C.c_uint64), ("max_count", C.c_uint64), ("total_kmers", C.c_uint64), ("max_records", C.c_uint64)]


class _GunzipParams(C.Structure):
    _fields_ = [("device", C.c_int32), ("reserved", C.c_uint32), ("max_in_bytes", C.c_uint64), ("max_out_bytes", C.c_uint64)]


# kmcb200_bgzf_member: one BGZF member of a call
BGZF_MEMBER = np.dtype([("in_off", "<u8"), ("out_off", "<u8"), ("in_bytes", "<u4"), ("isize", "<u4")])
BGZF_MIN_MEMBER = 28                                                    # header, empty deflate block, trailer


class BinFragment(C.Structure):
    """kmcb200_bin_fragment: one bin's share of a split batch."""
    _fields_ = [("byte_off", C.c_uint64), ("bytes", C.c_uint64), ("n_rec", C.c_uint64), ("n_super_kmers", C.c_uint64),
                ("pack0", C.c_uint32), ("n_packs", C.c_uint32)]


EXPORTS = [
    "kmcb200_create", "kmcb200_destroy", "kmcb200_last_error", "kmcb200_out_rec_bytes", "kmcb200_out_capacity", "kmcb200_lut_entries",
    "kmcb200_host_alloc", "kmcb200_host_free", "kmcb200_process_bin", "kmcb200_process_bin_multi", "kmcb200_submit_bin", "kmcb200_submit_bin_indexed", "kmcb200_wait_bin", "kmcb200_sort_records",
    "kmcb200_dev_process_bin", "kmcb200_dev_expand", "kmcb200_dev_sort", "kmcb200_dev_count", "kmcb200_kernel_launches",
    "kmcb200_stage_times", "kmcb200_stage_names", "kmcb200_leaf_plan",
    "kmcb200_wait_bin_scanned", "kmcb200_db_open", "kmcb200_db_last_error", "kmcb200_db_records", "kmcb200_db_reserve", "kmcb200_db_commit_bin", "kmcb200_db_close",
    "kmcb200_splitter_create", "kmcb200_splitter_destroy", "kmcb200_splitter_last_error", "kmcb200_split", "kmcb200_dev_split",
    "kmcb200_splitter_kernel_launches", "kmcb200_splitter_count_kxmers", "kmcb200_splitter_kxmer_totals",
    "kmcb200_splitter_set_homopolymer_compressed", "kmcb200_sigstats_set_homopolymer_compressed", "kmcb200_smallk_set_homopolymer_compressed",
    "kmcb200_sigstats_create", "kmcb200_sigstats_destroy", "kmcb200_sigstats_last_error", "kmcb200_sigstats_add", "kmcb200_dev_sigstats_add",
    "kmcb200_sigstats_read", "kmcb200_sigstats_reset", "kmcb200_sigstats_kernel_launches", "kmcb200_signature_map", "kmcb200_stage2_bin_order",
    "kmcb200_fastx_create", "kmcb200_fastx_destroy", "kmcb200_fastx_last_error", "kmcb200_fastx_kernel_launches", "kmcb200_fastx_parse",
    "kmcb200_fastx_last_records", "kmcb200_dev_fastx_parse", "kmcb200_split_fastx", "kmcb200_sigstats_add_fastx",
    "kmcb200_smallk_create", "kmcb200_smallk_destroy", "kmcb200_smallk_last_error", "kmcb200_smallk_kernel_launches", "kmcb200_smallk_add",
    "kmcb200_dev_smallk_add", "kmcb200_smallk_add_fastx", "kmcb200_smallk_read", "kmcb200_smallk_reset", "kmcb200_smallk_finish",
    "kmcb200_smallk_emit", "kmcb200_smallk_write_db",
    "kmcb200_estimator_create", "kmcb200_estimator_destroy", "kmcb200_estimator_last_error", "kmcb200_estimator_kernel_launches",
    "kmcb200_estimator_add", "kmcb200_dev_estimator_add", "kmcb200_estimator_add_fastx", "kmcb200_estimator_read",
    "kmcb200_estimator_histogram", "kmcb200_estimator_reset",
    "kmcb200_bgzf_scan", "kmcb200_gunzip_create", "kmcb200_gunzip_destroy", "kmcb200_gunzip_last_error", "kmcb200_gunzip_kernel_launches",
    "kmcb200_gunzip_inflate", "kmcb200_dev_gunzip_inflate",
    "kmcb200_kmcdb_create", "kmcb200_kmcdb_destroy", "kmcb200_kmcdb_last_error", "kmcb200_kmcdb_kernel_launches", "kmcb200_kmcdb_decode",
    "kmcb200_dev_kmcdb_decode", "kmcb200_split_kmcdb", "kmcb200_smallk_add_kmcdb", "kmcb200_estimator_add_kmcdb",
]

FASTQ, FASTA, BAM, BAM_ORIGINAL_STRAND = 1, 2, 4, 5                    # KMCB200_FASTQ / _FASTA / _BAM / _BAM_ORIGINAL_STRAND
FASTX_NO_LIMIT = (1 << 64) - 1

_lib = None


def load_library(build_if_needed=True):
    """Loads (building it first when nvcc is around and the sources are newer) the CUDA library. Fails loudly if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_needed and os.path.exists(_build.NVCC) and _build.needs_build():
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise KmcB200Error(ERR_NO_DEVICE, "%s is missing: run `python -m kmc_b200.build` (there is no CPU fallback)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int32
    L.kmcb200_create.argtypes = [C.POINTER(_Params), C.POINTER(vp)]
    L.kmcb200_destroy.argtypes = [vp]
    L.kmcb200_destroy.restype = None
    L.kmcb200_last_error.argtypes = [vp]
    L.kmcb200_last_error.restype = C.c_char_p
    L.kmcb200_out_rec_bytes.argtypes = [vp]
    L.kmcb200_out_rec_bytes.restype = u32
    L.kmcb200_out_capacity.argtypes = [vp, u64]
    L.kmcb200_out_capacity.restype = u64
    L.kmcb200_lut_entries.argtypes = [vp]
    L.kmcb200_lut_entries.restype = u64
    L.kmcb200_host_alloc.argtypes = [vp, u64, C.POINTER(vp)]
    L.kmcb200_host_free.argtypes = [vp, vp]
    L.kmcb200_process_bin.argtypes = [vp, i32, vp, u64, u64, u64, vp, vp, u32, vp, u64, C.POINTER(u64), vp, vp]
    L.kmcb200_process_bin_multi.argtypes = [vp, u32, i32, vp, u64, u64, vp, u32, vp, u64, C.POINTER(u64), vp, vp]
    L.kmcb200_submit_bin.argtypes = [vp, u32, i32, vp, u64, u64, u64, vp, vp, u32, vp, u64, vp]
    L.kmcb200_submit_bin_indexed.argtypes = [vp, u32, i32, vp, u64, u64, vp, u32, vp, u64, vp, vp, u64, vp]
    L.kmcb200_wait_bin.argtypes = [vp, u32, C.POINTER(u64), vp]
    L.kmcb200_sort_records.argtypes = [vp, vp, vp, u64, u32, u32]
    L.kmcb200_dev_process_bin.argtypes = [vp, u32, vp, u64, u64, vp, u32, vp, u64, vp, vp, vp]
    L.kmcb200_dev_expand.argtypes = [vp, u32, vp, u64, u64, vp, u32, vp, vp, vp]
    L.kmcb200_dev_sort.argtypes = [vp, u32, vp, vp, u64, u32, C.c_int, vp]
    L.kmcb200_dev_count.argtypes = [vp, u32, vp, u64, vp, u64, vp, vp, vp]
    L.kmcb200_kernel_launches.argtypes = [vp]
    L.kmcb200_kernel_launches.restype = u64
    L.kmcb200_stage_times.argtypes = [vp, u32, C.POINTER(C.c_float), u32]
    L.kmcb200_stage_names.argtypes = [vp, u32, C.c_char_p, u32]
    L.kmcb200_leaf_plan.argtypes = [vp, u32, C.POINTER(C.c_uint32)]
    L.kmcb200_wait_bin_scanned.argtypes = [vp, u32, u64, C.POINTER(u64), vp]
    L.kmcb200_db_open.argtypes = [C.POINTER(_DbParams), C.c_char_p, u64, C.POINTER(vp)]
    L.kmcb200_db_last_error.argtypes = [vp]
    L.kmcb200_db_last_error.restype = C.c_char_p
    L.kmcb200_db_records.argtypes = [vp]
    L.kmcb200_db_records.restype = u64
    L.kmcb200_db_reserve.argtypes = [vp, u64, C.POINTER(vp)]
    L.kmcb200_db_commit_bin.argtypes = [vp, u64, vp, C.c_int, vp, vp, u32]
    L.kmcb200_db_close.argtypes = [vp, vp]
    L.kmcb200_splitter_create.argtypes = [C.POINTER(_SplitParams), vp, C.POINTER(vp)]
    L.kmcb200_splitter_destroy.argtypes = [vp]
    L.kmcb200_splitter_destroy.restype = None
    L.kmcb200_splitter_last_error.argtypes = [vp]
    L.kmcb200_splitter_last_error.restype = C.c_char_p
    L.kmcb200_split.argtypes = [vp, vp, u64, vp, u64, C.POINTER(u64), vp, u64, C.POINTER(u64), vp]
    L.kmcb200_dev_split.argtypes = [vp, vp, u64, vp, u64, vp, u64, vp, vp, vp]
    L.kmcb200_splitter_kernel_launches.argtypes = [vp]
    L.kmcb200_splitter_kernel_launches.restype = u64
    L.kmcb200_splitter_count_kxmers.argtypes = [vp, C.c_int]
    L.kmcb200_splitter_kxmer_totals.argtypes = [vp, vp]
    L.kmcb200_splitter_set_homopolymer_compressed.argtypes = [vp, C.c_int]
    L.kmcb200_sigstats_set_homopolymer_compressed.argtypes = [vp, C.c_int]
    L.kmcb200_smallk_set_homopolymer_compressed.argtypes = [vp, C.c_int]
    L.kmcb200_sigstats_create.argtypes = [C.POINTER(_SigstatsParams), C.POINTER(vp)]
    L.kmcb200_sigstats_destroy.argtypes = [vp]
    L.kmcb200_sigstats_destroy.restype = None
    L.kmcb200_sigstats_last_error.argtypes = [vp]
    L.kmcb200_sigstats_last_error.restype = C.c_char_p
    L.kmcb200_sigstats_add.argtypes = [vp, vp, u64]
    L.kmcb200_dev_sigstats_add.argtypes = [vp, vp, u64, vp]
    L.kmcb200_sigstats_read.argtypes = [vp, vp]
    L.kmcb200_sigstats_reset.argtypes = [vp]
    L.kmcb200_sigstats_kernel_launches.argtypes = [vp]
    L.kmcb200_sigstats_kernel_launches.restype = u64
    L.kmcb200_signature_map.argtypes = [vp, u32, u32, vp]
    L.kmcb200_stage2_bin_order.argtypes = [u32, vp, vp, vp, u32, u32, u64, u64, u32, vp]
    L.kmcb200_fastx_create.argtypes = [C.POINTER(_FastxParams), C.POINTER(vp)]
    L.kmcb200_fastx_destroy.argtypes = [vp]
    L.kmcb200_fastx_destroy.restype = None
    L.kmcb200_fastx_last_error.argtypes = [vp]
    L.kmcb200_fastx_last_error.restype = C.c_char_p
    L.kmcb200_fastx_kernel_launches.argtypes = [vp]
    L.kmcb200_fastx_kernel_launches.restype = u64
    L.kmcb200_fastx_last_records.argtypes = [vp]
    L.kmcb200_fastx_last_records.restype = u64
    L.kmcb200_fastx_parse.argtypes = [vp, vp, u64, C.c_int, u64, vp, u64, C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_dev_fastx_parse.argtypes = [vp, vp, u64, C.c_int, u64, vp, u64, vp, vp]
    L.kmcb200_split_fastx.argtypes = [vp, vp, vp, u64, C.c_int, vp, u64, C.POINTER(u64), vp, u64, C.POINTER(u64), vp, C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_sigstats_add_fastx.argtypes = [vp, vp, vp, u64, C.c_int, u64, C.POINTER(u64)]
    L.kmcb200_smallk_create.argtypes = [C.POINTER(_SmallKParams), C.POINTER(vp)]
    L.kmcb200_smallk_destroy.argtypes = [vp]
    L.kmcb200_smallk_destroy.restype = None
    L.kmcb200_smallk_last_error.argtypes = [vp]
    L.kmcb200_smallk_last_error.restype = C.c_char_p
    L.kmcb200_smallk_kernel_launches.argtypes = [vp]
    L.kmcb200_smallk_kernel_launches.restype = u64
    L.kmcb200_smallk_add.argtypes = [vp, vp, u64]
    L.kmcb200_dev_smallk_add.argtypes = [vp, vp, u64, vp]
    L.kmcb200_smallk_add_fastx.argtypes = [vp, vp, vp, u64, C.c_int, C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_smallk_read.argtypes = [vp, vp]
    L.kmcb200_smallk_reset.argtypes = [vp]
    L.kmcb200_smallk_finish.argtypes = [vp, u32, u64, u64, C.POINTER(u32), C.POINTER(u32), C.POINTER(u64), vp]
    L.kmcb200_smallk_emit.argtypes = [vp, vp, u64, vp]
    L.kmcb200_smallk_write_db.argtypes = [vp, C.c_char_p, u32, u64, u64, vp]
    L.kmcb200_estimator_create.argtypes = [C.POINTER(_EstimatorParams), C.POINTER(vp)]
    L.kmcb200_estimator_destroy.argtypes = [vp]
    L.kmcb200_estimator_destroy.restype = None
    L.kmcb200_estimator_last_error.argtypes = [vp]
    L.kmcb200_estimator_last_error.restype = C.c_char_p
    L.kmcb200_estimator_kernel_launches.argtypes = [vp]
    L.kmcb200_estimator_kernel_launches.restype = u64
    L.kmcb200_estimator_add.argtypes = [vp, vp, u64]
    L.kmcb200_dev_estimator_add.argtypes = [vp, vp, u64, vp]
    L.kmcb200_estimator_add_fastx.argtypes = [vp, vp, vp, u64, C.c_int, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_estimator_read.argtypes = [vp, vp]
    L.kmcb200_estimator_histogram.argtypes = [vp, vp, u64, C.POINTER(u64)]
    L.kmcb200_estimator_reset.argtypes = [vp]
    L.kmcb200_bgzf_scan.argtypes = [vp, u64, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_gunzip_create.argtypes = [C.POINTER(_GunzipParams), C.POINTER(vp)]
    L.kmcb200_gunzip_destroy.argtypes = [vp]
    L.kmcb200_gunzip_destroy.restype = None
    L.kmcb200_gunzip_last_error.argtypes = [vp]
    L.kmcb200_gunzip_last_error.restype = C.c_char_p
    L.kmcb200_gunzip_kernel_launches.argtypes = [vp]
    L.kmcb200_gunzip_kernel_launches.restype = u64
    L.kmcb200_gunzip_inflate.argtypes = [vp, vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_dev_gunzip_inflate.argtypes = [vp, vp, u64, vp, u64, vp, u64, vp, vp]
    L.kmcb200_kmcdb_create.argtypes = [C.POINTER(_KmcDbParams), vp, u64, C.POINTER(vp)]
    L.kmcb200_kmcdb_destroy.argtypes = [vp]
    L.kmcb200_kmcdb_destroy.restype = None
    L.kmcb200_kmcdb_last_error.argtypes = [vp]
    L.kmcb200_kmcdb_last_error.restype = C.c_char_p
    L.kmcb200_kmcdb_kernel_launches.argtypes = [vp]
    L.kmcb200_kmcdb_kernel_launches.restype = u64
    L.kmcb200_kmcdb_decode.argtypes = [vp, vp, u64, u64, vp, u64, C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_dev_kmcdb_decode.argtypes = [vp, vp, u64, u64, vp, u64, vp, vp]
    L.kmcb200_split_kmcdb.argtypes = [vp, vp, vp, u64, u64, vp, u64, C.POINTER(u64), vp, u64, C.POINTER(u64), vp, C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_smallk_add_kmcdb.argtypes = [vp, vp, vp, u64, u64, C.POINTER(u64), C.POINTER(u64)]
    L.kmcb200_estimator_add_kmcdb.argtypes = [vp, vp, vp, u64, u64, C.POINTER(u64), C.POINTER(u64)]
    _lib = L
    return L


@dataclass
class Stage2Params:
    """The per-run parameters CKmerBinSorter takes from CKMCParams (kmc_core/kb_sorter.h:165-200)."""
    kmer_len: int = 31
    both_strands: bool = True
    cutoff_min: int = 2
    cutoff_max: int = 1_000_000_000
    counter_max: int = 255
    lut_prefix_len: int = 7


@dataclass
class SuperKmerBin:
    """One bin as stage 1 leaves it: byte stream + CBinDesc counters + expander packs (queues.h:376-679)."""
    data: np.ndarray            # uint8
    n_rec: int
    pack_bytes: np.ndarray      # uint64
    n_super_kmers: int = 0
    kmer_len: int = 31

    @property
    def size(self):
        return int(self.data.size)


@dataclass
class BinResult:
    """What CKmerBinSorter hands to CKmerQueue::push (queues.h:826): emitted records, raw LUT, the four counters."""
    payload: np.ndarray         # uint8, concatenated (suffix, counter) records
    lut: np.ndarray             # uint64[4^p]
    n_unique: int
    n_cutoff_min: int
    n_cutoff_max: int
    n_total: int

    @property
    def stats(self):
        return (self.n_unique, self.n_cutoff_min, self.n_cutoff_max, self.n_total)


class _Handle:
    """One handle of the C ABI: the symbols <_prefix>_<_create> / _destroy / _last_error, create-or-raise, error check, close."""
    _prefix = None
    _create = "create"

    def _sym(self, name):
        return getattr(self.lib, "%s_%s" % (self._prefix, name))

    def _open(self, *args):
        """The family's create call on `args`; its handle pointer is the last argument."""
        self.lib = load_library()
        self._h = C.c_void_p(None)
        rc = self._sym(self._create)(*args, C.byref(self._h))
        if rc != 0:
            raise KmcB200Error(rc, (self._sym("last_error")(None) or b"").decode())

    def _check(self, rc):
        if rc < 0:
            raise KmcB200Error(rc, (self._sym("last_error")(self._h) or b"").decode())
        return rc

    def close(self):
        if self._h:
            self._sym("destroy")(self._h)
            self._h = C.c_void_p(None)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Stage2Context(_Handle):
    """One GPU's stage-2 engine (one per sorter thread in KMC terms)."""
    _prefix = "kmcb200"

    def __init__(self, params: Stage2Params, device=0, n_slots=1):
        self.params = params
        p = _Params(params.kmer_len, int(params.both_strands), params.cutoff_min, min(params.cutoff_max, 0xFFFFFFFF),
                    min(params.counter_max, 0xFFFFFFFF), params.lut_prefix_len, device, n_slots)
        self._open(C.byref(p))
        self.device = device
        self.n_slots = n_slots
        self.words = (params.kmer_len + 31) // 32
        self.key_bytes = (params.kmer_len + 3) // 4
        self.out_rec_bytes = self.lib.kmcb200_out_rec_bytes(self._h)
        self.lut_entries = self.lib.kmcb200_lut_entries(self._h)

    def out_capacity(self, n_rec):
        return int(self.lib.kmcb200_out_capacity(self._h, n_rec))

    def kernel_launches(self):
        return int(self.lib.kmcb200_kernel_launches(self._h))

    def stage_times(self, slot=0):
        ms = (C.c_float * 48)()
        n = self._check(self.lib.kmcb200_stage_times(self._h, slot, ms, 48))
        names = C.create_string_buffer(2048)
        self._check(self.lib.kmcb200_stage_names(self._h, slot, names, 2048))
        nm = names.value.decode().split(",") if names.value else []
        return {"expand_ms": ms[0], "sort_ms": ms[1], "count_ms": ms[2], "pass_ms": [ms[3 + i] for i in range(n)], "pass_names": nm}

    LEAF_KERNELS = {0: None, 1: "hash", 2: "cta", 3: "wide"}

    def leaf_plan(self, slot=0):
        """How the slot's last bin counted its leaves: (bits of the second partition level, leaf kernel: "hash" = leaf_hash_kernel,
        "cta" = leaf_hash_cta_kernel, "wide" = leaf_hash_wide_kernel, None = the leaves were sorted)."""
        out = (C.c_uint32 * 2)()
        self._check(self.lib.kmcb200_leaf_plan(self._h, slot, out))
        return int(out[0]), self.LEAF_KERNELS[int(out[1])]

    # -- seam #2, host buffers
    def process_bin(self, b: SuperKmerBin, out=None, lut=None, bin_id=0) -> BinResult:
        cap = self.out_capacity(b.n_rec) + 64
        out = np.empty(cap, dtype=np.uint8) if out is None else out
        lut = np.empty(self.lut_entries, dtype=np.uint64) if lut is None else lut
        stats = (C.c_uint64 * 4)()
        nbytes = C.c_uint64(0)
        data = np.ascontiguousarray(b.data)
        packs = np.ascontiguousarray(b.pack_bytes, dtype=np.uint64)
        self._check(self.lib.kmcb200_process_bin(self._h, bin_id, data.ctypes.data, data.size, b.n_rec, b.n_rec, packs.ctypes.data, None, packs.size,
                                                 out.ctypes.data, out.size, C.byref(nbytes), lut.ctypes.data, stats))
        return BinResult(out[:nbytes.value], lut, *[int(x) for x in stats])

    def submit_bin(self, slot, data_ptr, size, n_rec, packs: np.ndarray, out_ptr, out_capacity, lut_ptr, bin_id=0):
        self._check(self.lib.kmcb200_submit_bin(self._h, slot, bin_id, data_ptr, size, n_rec, n_rec, packs.ctypes.data, None, packs.size,
                                                out_ptr, out_capacity, lut_ptr))

    def submit_bin_indexed(self, slot, data_ptr, size, n_rec, packs: np.ndarray, extras: np.ndarray, pack_superkmers: np.ndarray, out_ptr, out_capacity, lut_ptr, bin_id=0):
        """submit_bin with stage 1's length bytes as a separate array (N4: no record walk on the GPU)."""
        extras = np.ascontiguousarray(extras, dtype=np.uint8)
        psk = np.ascontiguousarray(pack_superkmers, dtype=np.uint32)
        self._keep = (extras, psk)
        self._check(self.lib.kmcb200_submit_bin_indexed(self._h, slot, bin_id, data_ptr, size, n_rec, packs.ctypes.data, packs.size,
                                                        extras.ctypes.data, extras.size, psk.ctypes.data, out_ptr, out_capacity, lut_ptr))

    def wait_bin_scanned(self, slot, lut_base):
        """wait_bin with the LUT already prefix-summed on the GPU and offset by lut_base (what goes into .kmc_pre)."""
        stats = (C.c_uint64 * 4)()
        nbytes = C.c_uint64(0)
        self._check(self.lib.kmcb200_wait_bin_scanned(self._h, slot, lut_base, C.byref(nbytes), stats))
        return int(nbytes.value), tuple(int(x) for x in stats)

    def wait_bin(self, slot):
        stats = (C.c_uint64 * 4)()
        nbytes = C.c_uint64(0)
        self._check(self.lib.kmcb200_wait_bin(self._h, slot, C.byref(nbytes), stats))
        return int(nbytes.value), tuple(int(x) for x in stats)

    @staticmethod
    def process_bin_multi(ctxs, b: "SuperKmerBin", out=None, lut=None) -> "BinResult":
        """One bin split over several contexts / GPUs by key range (kmcb200_process_bin_multi)."""
        c0 = ctxs[0]
        cap = c0.out_capacity(b.n_rec) + 64
        out = np.empty(cap, dtype=np.uint8) if out is None else out
        lut = np.empty(c0.lut_entries, dtype=np.uint64) if lut is None else lut
        stats = (C.c_uint64 * 4)()
        nbytes = C.c_uint64(0)
        data = np.ascontiguousarray(b.data)
        packs = np.ascontiguousarray(b.pack_bytes, dtype=np.uint64)
        arr = (C.c_void_p * len(ctxs))(*[c._h for c in ctxs])
        c0._check(c0.lib.kmcb200_process_bin_multi(arr, len(ctxs), 0, data.ctypes.data, data.size, b.n_rec, packs.ctypes.data, packs.size,
                                                   out.ctypes.data, out.size, C.byref(nbytes), lut.ctypes.data, stats))
        return BinResult(out[:nbytes.value], lut, *[int(x) for x in stats])

    # -- seam #1
    def sort_records(self, recs: np.ndarray, key_bytes=None):
        """recs: uint64 [n, words].  Returns the sorted copy (SortFunction contract, raduls.h:19-20)."""
        recs = np.ascontiguousarray(recs, dtype=np.uint64).copy()
        n, w = recs.shape
        tmp = np.empty_like(recs)
        kb = self.key_bytes if key_bytes is None else key_bytes
        where = self._check(self.lib.kmcb200_sort_records(self._h, recs.ctypes.data, tmp.ctypes.data, n, 8 * w, kb))
        return tmp if where == 1 else recs

    # -- device-level (pointers are device pointers: ints or torch tensors' data_ptr())
    def dev_process_bin(self, slot, d_bin, size, n_rec, packs: np.ndarray, d_out, out_capacity, d_lut, d_result, stream=None):
        packs = np.ascontiguousarray(packs, dtype=np.uint64)
        self._check(self.lib.kmcb200_dev_process_bin(self._h, slot, d_bin, size, n_rec, packs.ctypes.data, packs.size, d_out, out_capacity, d_lut, d_result, stream))

    def dev_expand(self, slot, d_bin, size, n_rec, packs: np.ndarray, d_recs, d_result=None, stream=None):
        packs = np.ascontiguousarray(packs, dtype=np.uint64)
        self._check(self.lib.kmcb200_dev_expand(self._h, slot, d_bin, size, n_rec, packs.ctypes.data, packs.size, d_recs, d_result, stream))

    def dev_sort(self, slot, d_recs, d_tmp, n, key_bytes=None, hist_ready=False, stream=None):
        return self._check(self.lib.kmcb200_dev_sort(self._h, slot, d_recs, d_tmp, n, self.key_bytes if key_bytes is None else key_bytes, int(hist_ready), stream))

    def dev_count(self, slot, d_sorted, n, d_out, out_capacity, d_lut, d_result, stream=None):
        self._check(self.lib.kmcb200_dev_count(self._h, slot, d_sorted, n, d_out, out_capacity, d_lut, d_result, stream))


class DbWriter(_Handle):
    """KMC database files from per-bin results (kmcb200_db_*): pinned staging ring + writer thread; format of kb_completer.cpp:59-326."""
    _prefix = "kmcb200_db"
    _create = "open"

    def __init__(self, path_prefix, kmer_len, counter_size, lut_prefix_len, signature_len, cutoff_min, cutoff_max, both_strands, staging_bytes=1 << 28):
        p = _DbParams(kmer_len, counter_size, lut_prefix_len, signature_len, cutoff_min, min(cutoff_max, 0xFFFFFFFF), int(both_strands))
        self._open(C.byref(p), path_prefix.encode(), staging_bytes)
        self.lut_entries = 1 << (2 * lut_prefix_len)

    @property
    def records(self):
        return int(self.lib.kmcb200_db_records(self._h))

    def reserve(self, nbytes):
        ptr = C.c_void_p(None)
        self._check(self.lib.kmcb200_db_reserve(self._h, nbytes, C.byref(ptr)))
        return ptr.value

    def commit_bin(self, payload_bytes, lut: np.ndarray, stats, signatures=(), raw_lut=False):
        lut = np.ascontiguousarray(lut, dtype=np.uint64)
        assert lut.size == self.lut_entries
        st = (C.c_uint64 * 4)(*[int(x) for x in stats])
        sig = np.ascontiguousarray(np.asarray(signatures, dtype=np.uint32))
        self._check(self.lib.kmcb200_db_commit_bin(self._h, payload_bytes, lut.ctypes.data, int(raw_lut), st, sig.ctypes.data if sig.size else None, sig.size))

    def close(self):
        tot = (C.c_uint64 * 4)()
        h, self._h = self._h, C.c_void_p(None)
        rc = self.lib.kmcb200_db_close(h, tot)
        if rc != 0:
            raise KmcB200Error(rc, "kmcb200_db_close")
        return tuple(int(x) for x in tot)

    def __del__(self):          # only close() ends a database: a writer that is dropped leaves its files unfinished
        pass


class Splitter(_Handle):
    """Stage 1 on one GPU (kmcb200_splitter_*): batches of sequences -> KMC bins (CSplitter::ProcessReads, kmc_core/splitter.cpp:557-677).

    A batch is one byte array in which every byte other than ACGTacgt separates (reads.sequences_to_batch makes one from FASTQ / FASTA).
    `signature_map` has 4^signature_len + 1 entries, each below n_bins.  homopolymer_compressed: every batch is homopolymer-compressed on
    the GPU first, as `kmc -hc` does (see set_homopolymer_compressed)."""
    _prefix = "kmcb200_splitter"

    def __init__(self, kmer_len, signature_len, signature_map, n_bins=None, device=0, max_batch_bytes=1 << 26, homopolymer_compressed=False):
        sig_map = np.ascontiguousarray(signature_map, dtype=np.uint32)
        if sig_map.size != (1 << (2 * signature_len)) + 1:
            raise KmcB200Error(ERR_INVALID, "signature_map has %d entries, 4^%d + 1 expected" % (sig_map.size, signature_len))
        self.n_bins = int(sig_map.max()) + 1 if n_bins is None else int(n_bins)
        self.kmer_len, self.signature_len, self.max_batch_bytes = kmer_len, signature_len, max_batch_bytes
        p = _SplitParams(kmer_len, signature_len, self.n_bins, device, max_batch_bytes)
        self._open(C.byref(p), sig_map.ctypes.data)
        self._out = np.empty(0, dtype=np.uint8)
        self._packs = np.empty(0, dtype=np.uint64)
        if homopolymer_compressed:
            self.set_homopolymer_compressed(True)

    def kernel_launches(self):
        return int(self.lib.kmcb200_splitter_kernel_launches(self._h))

    def split_raw(self, batch, out=None, pack_bytes=None):
        """kmcb200_split into the given (or internal, grown as needed) buffers: (out[:bytes], pack_bytes[:n_packs], fragments)."""
        seq = np.ascontiguousarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)
        frags = (BinFragment * self.n_bins)()
        nbytes, npacks = C.c_uint64(0), C.c_uint64(0)
        own = out is None
        for _ in range(2):
            o = self._out if own else out
            pk = self._packs if pack_bytes is None else pack_bytes
            rc = self.lib.kmcb200_split(self._h, seq.ctypes.data, seq.size, o.ctypes.data, o.size, C.byref(nbytes),
                                        pk.ctypes.data, pk.size, C.byref(npacks), frags)
            if rc == ERR_CAPACITY and own and pack_bytes is None:
                self._out = np.empty(int(nbytes.value * 1.25) + 1024, dtype=np.uint8)
                self._packs = np.empty(int(npacks.value * 1.25) + 64, dtype=np.uint64)
                continue
            self._check(rc)
            return o[:nbytes.value], pk[:npacks.value], list(frags)
        raise KmcB200Error(ERR_CAPACITY, "kmcb200_split: buffers still too small")

    def split(self, batch):
        """One batch -> one SuperKmerBin fragment per bin (copies; empty bins have size 0)."""
        out, packs, frags = self.split_raw(batch)
        res = []
        for f in frags:
            res.append(SuperKmerBin(data=out[f.byte_off:f.byte_off + f.bytes].copy(), n_rec=int(f.n_rec),
                                    pack_bytes=packs[f.pack0:f.pack0 + f.n_packs].copy(), n_super_kmers=int(f.n_super_kmers), kmer_len=self.kmer_len))
        return res

    def dev_split(self, d_seq, nbytes, d_out, out_capacity, d_pack_bytes, pack_capacity, d_frags, d_result, stream=None):
        """kmcb200_dev_split: device pointers (ints or tensors' data_ptr()); d_frags holds n_bins x 40 bytes, d_result 5 x uint64."""
        self._check(self.lib.kmcb200_dev_split(self._h, d_seq, nbytes, d_out, out_capacity, d_pack_bytes, pack_capacity, d_frags, d_result, stream))

    def split_fastx(self, parser, raw, is_final=True):
        """kmcb200_split_fastx: a raw FASTQ / FASTA chunk (bytes or a uint8 array, ideally pinned) parsed on the GPU by `parser` straight into
        this splitter's batch buffer, then split like split_raw.  Returns (out[:bytes], pack_bytes[:n_packs], fragments, consumed, seq_bytes):
        a non-final chunk is parsed up to its last record end, and the caller carries raw[consumed:] into the next chunk."""
        a = _as_u8(raw)
        frags = (BinFragment * self.n_bins)()
        nbytes, npacks, consumed, seq_bytes = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        for _ in range(2):
            rc = self.lib.kmcb200_split_fastx(self._h, parser._h, a.ctypes.data, a.size, int(bool(is_final)), self._out.ctypes.data, self._out.size,
                                              C.byref(nbytes), self._packs.ctypes.data, self._packs.size, C.byref(npacks), frags, C.byref(consumed),
                                              C.byref(seq_bytes))
            if rc == ERR_CAPACITY:
                self._out = np.empty(int(nbytes.value * 1.25) + 1024, dtype=np.uint8)
                self._packs = np.empty(int(npacks.value * 1.25) + 64, dtype=np.uint64)
                continue
            self._check(rc)
            return self._out[:nbytes.value], self._packs[:npacks.value], list(frags), int(consumed.value), int(seq_bytes.value)
        raise KmcB200Error(ERR_CAPACITY, "kmcb200_split_fastx: buffers still too small")

    def split_kmcdb(self, decoder, suffix, first_record):
        """kmcb200_split_kmcdb: whole .kmc_suf records (bytes or a uint8 array, ideally pinned; first_record the index of the first) decoded
        on the GPU by `decoder` (a KmcDbDecoder) straight into this splitter's batch buffer, then split like split_raw.  Returns
        (out[:bytes], pack_bytes[:n_packs], fragments, seq_bytes, kept)."""
        a = _as_u8(suffix)
        n = decoder.records_in(a)
        frags = (BinFragment * self.n_bins)()
        nbytes, npacks, seq_bytes, kept = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        for _ in range(2):
            rc = self.lib.kmcb200_split_kmcdb(self._h, decoder._h, a.ctypes.data, n, int(first_record), self._out.ctypes.data, self._out.size,
                                              C.byref(nbytes), self._packs.ctypes.data, self._packs.size, C.byref(npacks), frags,
                                              C.byref(seq_bytes), C.byref(kept))
            if rc == ERR_CAPACITY:
                self._out = np.empty(int(nbytes.value * 1.25) + 1024, dtype=np.uint8)
                self._packs = np.empty(int(npacks.value * 1.25) + 64, dtype=np.uint64)
                continue
            self._check(rc)
            decoder.last_kept = int(kept.value)
            return self._out[:nbytes.value], self._packs[:npacks.value], list(frags), int(seq_bytes.value), int(kept.value)
        raise KmcB200Error(ERR_CAPACITY, "kmcb200_split_kmcdb: buffers still too small")

    def count_kxmers(self, both_strands=True):
        """From now on every split also counts, per bin, the collector's (k+x)-mers (n_plus_x_recs); zeroes the totals."""
        self._check(self.lib.kmcb200_splitter_count_kxmers(self._h, int(bool(both_strands))))

    def set_homopolymer_compressed(self, on=True):
        """kmcb200_splitter_set_homopolymer_compressed: while on, every batch (host, device twin or parsed chunk) has each run of one base
        collapsed to a single base on the GPU before it is split, as `kmc -hc` does; 3 more kernel launches per batch and
        max_batch_bytes more bytes of HBM, allocated the first time it is turned on."""
        self._check(self.lib.kmcb200_splitter_set_homopolymer_compressed(self._h, int(bool(on))))

    def kxmer_totals(self):
        """uint64[n_bins]: the (k+x)-mers per bin since count_kxmers (zeros for k % 32 == 0, where stage 2 sorts plain k-mers)."""
        out = np.zeros(self.n_bins, dtype=np.uint64)
        self._check(self.lib.kmcb200_splitter_kxmer_totals(self._h, out.ctypes.data))
        return out


class SignatureStats(_Handle):
    """Stage 0 on one GPU (kmcb200_sigstats_*): k-mers per signature over batches of sequences, what CSplitter::CalcStats counts
    (kmc_core/splitter.cpp:439-533).  Batches as for Splitter; the counts (uint32[4^signature_len + 1]) add up until reset().
    homopolymer_compressed as for Splitter."""
    _prefix = "kmcb200_sigstats"

    def __init__(self, kmer_len, signature_len, device=0, max_batch_bytes=1 << 26, homopolymer_compressed=False):
        self.kmer_len, self.signature_len, self.max_batch_bytes = kmer_len, signature_len, max_batch_bytes
        p = _SigstatsParams(kmer_len, signature_len, device, 0, max_batch_bytes)
        self._open(C.byref(p))
        if homopolymer_compressed:
            self.set_homopolymer_compressed(True)

    def set_homopolymer_compressed(self, on=True):
        """kmcb200_sigstats_set_homopolymer_compressed: while on, every batch (host, device twin or parsed chunk) has each run of one base
        collapsed to a single base on the GPU before it is counted, as `kmc -hc` does; 3 more kernel launches per batch and
        max_batch_bytes more bytes of HBM, allocated the first time it is turned on."""
        self._check(self.lib.kmcb200_sigstats_set_homopolymer_compressed(self._h, int(bool(on))))

    def kernel_launches(self):
        return int(self.lib.kmcb200_sigstats_kernel_launches(self._h))

    def add(self, batch):
        seq = np.ascontiguousarray(np.frombuffer(batch, dtype=np.uint8) if isinstance(batch, (bytes, bytearray)) else batch, dtype=np.uint8)
        self._check(self.lib.kmcb200_sigstats_add(self._h, seq.ctypes.data, seq.size))

    def dev_add(self, d_seq, nbytes, stream=None):
        """kmcb200_dev_sigstats_add: d_seq a device pointer (int or a tensor's data_ptr()), queued on `stream` (a cudaStream_t)."""
        self._check(self.lib.kmcb200_dev_sigstats_add(self._h, d_seq, nbytes, stream))

    def add_fastx(self, parser, raw, is_final=True, limit=None):
        """kmcb200_sigstats_add_fastx: a raw FASTQ / FASTA chunk parsed on the GPU by `parser` and counted.  With `limit`, only the records that
        start before raw[limit] are parsed.  Returns `consumed`, the bytes parsed (the caller carries the rest into its next chunk)."""
        a = _as_u8(raw)
        consumed = C.c_uint64(0)
        self._check(self.lib.kmcb200_sigstats_add_fastx(self._h, parser._h, a.ctypes.data, a.size, int(bool(is_final)),
                                                        FASTX_NO_LIMIT if limit is None else int(limit), C.byref(consumed)))
        return int(consumed.value)

    def read(self):
        out = np.zeros((1 << (2 * self.signature_len)) + 1, dtype=np.uint32)
        self._check(self.lib.kmcb200_sigstats_read(self._h, out.ctypes.data))
        return out

    def reset(self):
        self._check(self.lib.kmcb200_sigstats_reset(self._h))


class SmallKCounter(_Handle):
    """Small k (1..13) on one GPU (kmcb200_smallk_*), KMC's small-k mode (kmc_core/kmc.h:677-960): every k-mer of the batches counted in
    a direct array of 4^k uint64 counters (CSplitter::ProcessReadsSmallK), then a KMC1-format database (CSmallKCompleter).  Batches as for
    Splitter; the counts add up until reset().  There are no bins, so no signature length, map or caller-chosen LUT prefix length: finish()
    picks the LUT prefix length as the reference does.  homopolymer_compressed as for Splitter."""
    _prefix = "kmcb200_smallk"

    def __init__(self, kmer_len, both_strands=True, device=0, max_batch_bytes=1 << 26, homopolymer_compressed=False):
        self.kmer_len, self.both_strands, self.max_batch_bytes = kmer_len, bool(both_strands), max_batch_bytes
        p = _SmallKParams(kmer_len, int(bool(both_strands)), device, 0, max_batch_bytes)
        self._open(C.byref(p))
        if homopolymer_compressed:
            self.set_homopolymer_compressed(True)

    def set_homopolymer_compressed(self, on=True):
        """kmcb200_smallk_set_homopolymer_compressed: while on, every batch (host, device twin or parsed chunk) has each run of one base
        collapsed to a single base on the GPU before it is counted, as `kmc -hc` does; 3 more kernel launches per batch and
        max_batch_bytes more bytes of HBM, allocated the first time it is turned on."""
        self._check(self.lib.kmcb200_smallk_set_homopolymer_compressed(self._h, int(bool(on))))

    def kernel_launches(self):
        return int(self.lib.kmcb200_smallk_kernel_launches(self._h))

    def add(self, batch):
        seq = _as_u8(batch)
        self._check(self.lib.kmcb200_smallk_add(self._h, seq.ctypes.data, seq.size))

    def dev_add(self, d_seq, nbytes, stream=None):
        """kmcb200_dev_smallk_add: d_seq a device pointer (int or a tensor's data_ptr()), queued on `stream` (a cudaStream_t)."""
        self._check(self.lib.kmcb200_dev_smallk_add(self._h, d_seq, nbytes, stream))

    def add_fastx(self, parser, raw, is_final=True):
        """kmcb200_smallk_add_fastx: a raw FASTQ / FASTA chunk parsed on the GPU by `parser` and counted.  Returns `consumed`, the bytes
        parsed (the caller carries the rest into its next chunk); the length of the batch the chunk gave is left in last_seq_bytes."""
        a = _as_u8(raw)
        consumed, seq_bytes = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.kmcb200_smallk_add_fastx(self._h, parser._h, a.ctypes.data, a.size, int(bool(is_final)), C.byref(consumed),
                                                      C.byref(seq_bytes)))
        self.last_seq_bytes = int(seq_bytes.value)
        return int(consumed.value)

    def add_kmcdb(self, decoder, suffix, first_record):
        """kmcb200_smallk_add_kmcdb: whole .kmc_suf records decoded on the GPU by `decoder` (a KmcDbDecoder) and counted.  Returns the
        records kept; the batch's length is left in last_seq_bytes."""
        a = _as_u8(suffix)
        seq_bytes, kept = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.kmcb200_smallk_add_kmcdb(self._h, decoder._h, a.ctypes.data, decoder.records_in(a), int(first_record),
                                                      C.byref(seq_bytes), C.byref(kept)))
        self.last_seq_bytes = decoder.last_seq_bytes = int(seq_bytes.value)
        decoder.last_kept = int(kept.value)
        return decoder.last_kept

    def read(self):
        """uint64[4^k]: the counts of every k-mer value so far."""
        out = np.zeros(1 << (2 * self.kmer_len), dtype=np.uint64)
        self._check(self.lib.kmcb200_smallk_read(self._h, out.ctypes.data))
        return out

    def reset(self):
        self._check(self.lib.kmcb200_smallk_reset(self._h))

    def finish(self, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255):
        """kmcb200_smallk_finish: (lut_prefix_len, counter_size, suffix_bytes, (n_unique, n_cutoff_min, n_cutoff_max, n_total))."""
        lp, cs, nbytes = C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
        st = (C.c_uint64 * 4)()
        self._check(self.lib.kmcb200_smallk_finish(self._h, cutoff_min, min(int(cutoff_max), (1 << 64) - 1), min(int(counter_max), (1 << 64) - 1),
                                                   C.byref(lp), C.byref(cs), C.byref(nbytes), st))
        self._layout = (int(lp.value), int(nbytes.value))
        return int(lp.value), int(cs.value), int(nbytes.value), tuple(int(x) for x in st)

    def emit(self, out=None):
        """kmcb200_smallk_emit after finish(): (records, lut).  `out` (uint8, default: exactly suffix_bytes fresh bytes) receives the records;
        a shorter one raises ERR_CAPACITY and is left untouched."""
        lp, nbytes = getattr(self, "_layout", (0, 0))
        o = np.empty(nbytes, dtype=np.uint8) if out is None else out
        lut = np.empty(1 << (2 * lp), dtype=np.uint64)
        self._check(self.lib.kmcb200_smallk_emit(self._h, o.ctypes.data if o.size else None, o.size, lut.ctypes.data))
        return o[:nbytes], lut

    def write_db(self, path_prefix, cutoff_min=2, cutoff_max=1_000_000_000, counter_max=255):
        """kmcb200_smallk_write_db: path_prefix.kmc_pre / .kmc_suf in KMC1 format; returns (n_unique, n_cutoff_min, n_cutoff_max, n_total)."""
        tot = (C.c_uint64 * 4)()
        self._check(self.lib.kmcb200_smallk_write_db(self._h, path_prefix.encode(), cutoff_min, min(int(cutoff_max), (1 << 64) - 1),
                                                     min(int(counter_max), (1 << 64) - 1), tot))
        return tuple(int(x) for x in tot)


class HistogramEstimator(_Handle):
    """KMC's histogram estimator on one GPU (kmcb200_estimator_*), what `kmc -e` and `kmc --opt-out-size` run (CntHashEstimator,
    kmc_core/libs/ntHash/ntHashWrapper.h): the canonical ntHash of every k-mer (1 <= k <= 256) of the batches, sampled into two tables of
    2^27 uint32 counters with s = 7 or 11; histogram() is the reference's estimate of the k-mer count histogram.  Batches as for Splitter;
    the counters add up until reset().  The handle holds 1 GiB of counters on the device."""
    _prefix = "kmcb200_estimator"
    TABLE = 1 << 27

    def __init__(self, kmer_len, s=7, device=0, max_batch_bytes=1 << 26):
        self.kmer_len, self.s, self.max_batch_bytes = kmer_len, s, max_batch_bytes
        p = _EstimatorParams(kmer_len, s, device, 0, max_batch_bytes)
        self._open(C.byref(p))

    def kernel_launches(self):
        return int(self.lib.kmcb200_estimator_kernel_launches(self._h))

    def add(self, batch):
        seq = _as_u8(batch)
        self._check(self.lib.kmcb200_estimator_add(self._h, seq.ctypes.data, seq.size))

    def dev_add(self, d_seq, nbytes, stream=None):
        """kmcb200_dev_estimator_add: d_seq a device pointer (int or a tensor's data_ptr()), queued on `stream` (a cudaStream_t)."""
        self._check(self.lib.kmcb200_dev_estimator_add(self._h, d_seq, nbytes, stream))

    def add_fastx(self, parser, raw, is_final=True):
        """kmcb200_estimator_add_fastx: a raw FASTQ / FASTA chunk parsed on the GPU by `parser` and hashed.  Returns `consumed`, the bytes
        parsed (the caller carries the rest into its next chunk); the batch's length and the records parsed are left in last_seq_bytes and
        last_records."""
        a = _as_u8(raw)
        consumed, seq_bytes, recs = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.kmcb200_estimator_add_fastx(self._h, parser._h, a.ctypes.data, a.size, int(bool(is_final)), C.byref(consumed),
                                                         C.byref(seq_bytes), C.byref(recs)))
        self.last_seq_bytes, self.last_records = int(seq_bytes.value), int(recs.value)
        return int(consumed.value)

    def add_kmcdb(self, decoder, suffix, first_record):
        """kmcb200_estimator_add_kmcdb: whole .kmc_suf records decoded on the GPU by `decoder` (a KmcDbDecoder) and hashed.  Returns the
        records kept; the batch's length is left in last_seq_bytes."""
        a = _as_u8(suffix)
        seq_bytes, kept = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.kmcb200_estimator_add_kmcdb(self._h, decoder._h, a.ctypes.data, decoder.records_in(a), int(first_record),
                                                         C.byref(seq_bytes), C.byref(kept)))
        self.last_seq_bytes = decoder.last_seq_bytes = int(seq_bytes.value)
        decoder.last_kept = int(kept.value)
        return decoder.last_kept

    def read(self):
        """uint32[2, 2^27]: the two counter tables."""
        out = np.zeros((2, self.TABLE), dtype=np.uint32)
        self._check(self.lib.kmcb200_estimator_read(self._h, out.ctypes.data))
        return out

    def histogram(self):
        """uint64[max_occ + 1]: entry i estimates the distinct k-mers that occur i times (entry 0 is 0), as `kmc -e` writes it."""
        out = np.zeros(65537, dtype=np.uint64)
        n = C.c_uint64(0)
        self._check(self.lib.kmcb200_estimator_histogram(self._h, out.ctypes.data, out.size, C.byref(n)))
        return out[:n.value].copy()

    def reset(self):
        self._check(self.lib.kmcb200_estimator_reset(self._h))


def _as_u8(raw):
    return np.ascontiguousarray(np.frombuffer(raw, dtype=np.uint8) if isinstance(raw, (bytes, bytearray, memoryview)) else raw, dtype=np.uint8)


class FastxParser(_Handle):
    """Reads text -> batch on one GPU (kmcb200_fastx_*): raw FASTQ or FASTA chunks become the batches Splitter and SignatureStats take,
    byte for byte what kmc_b200.reads.sequences_to_batch makes of the whole file.  `fmt` is FASTQ / FASTA (or "fastq" / "fasta"): the
    caller's choice, by the first byte of the file's first non-empty line.  With BAM / BAM_ORIGINAL_STRAND (or "bam" / "bam_original_strand")
    chunks are decompressed BAM record bytes, the header skipped, and the batch is kmc_b200.reads.bam_records_to_batch's (original_strand
    for BAM_ORIGINAL_STRAND); a final chunk that ends inside a record and a malformed record raise ERR_INVALID.

    A chunk is parsed up to its last record end unless it is final (then to its end, as if it ended in '\n'); `consumed` says where the
    next chunk must start.  A record longer than the chunk is an error: since the limit here is raw bytes per chunk, a FASTQ record of more
    than about max_chunk_bytes / 2 bases cannot be parsed, where the host path (sequences_to_batch + batches) accepts sequences up to the
    batch size."""
    _prefix = "kmcb200_fastx"

    def __init__(self, fmt, device=0, max_chunk_bytes=1 << 26):
        self.format = {"fastq": FASTQ, "fasta": FASTA, "bam": BAM, "bam_original_strand": BAM_ORIGINAL_STRAND}.get(fmt, fmt) \
            if isinstance(fmt, str) else int(fmt)
        self.max_chunk_bytes = max_chunk_bytes
        p = _FastxParams(device, self.format, max_chunk_bytes)
        self._open(C.byref(p))

    def kernel_launches(self):
        return int(self.lib.kmcb200_fastx_kernel_launches(self._h))

    def last_records(self):
        """kmcb200_fastx_last_records: the records the latest host-buffer call parsed (parse or any handle's _fastx entry point)."""
        return int(self.lib.kmcb200_fastx_last_records(self._h))

    def parse(self, raw, is_final=True, limit=None, out=None):
        """kmcb200_fastx_parse: (batch, consumed).  `out` (uint8, default: bytes + 1 fresh bytes) receives the batch; a shorter one than the
        batch raises ERR_CAPACITY and is left untouched."""
        a = _as_u8(raw)
        o = np.empty(a.size + 1, dtype=np.uint8) if out is None else out
        consumed, nbytes = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.kmcb200_fastx_parse(self._h, a.ctypes.data, a.size, int(bool(is_final)), FASTX_NO_LIMIT if limit is None else int(limit),
                                                 o.ctypes.data, o.size, C.byref(consumed), C.byref(nbytes)))
        return o[:nbytes.value], int(consumed.value)

    def dev_parse(self, d_raw, nbytes, is_final, limit, d_seq, seq_capacity, d_result, stream=None):
        """kmcb200_dev_fastx_parse: device pointers (ints or tensors' data_ptr()); seq_capacity >= nbytes + 1; d_result receives 4 x uint64:
        consumed, sequence bytes, records, error (1: a non-final chunk without a record end; BAM: 2 truncated, 3 malformed)."""
        self._check(self.lib.kmcb200_dev_fastx_parse(self._h, d_raw, nbytes, int(bool(is_final)), FASTX_NO_LIMIT if limit is None else int(limit),
                                                     d_seq, seq_capacity, d_result, stream))


class KmcDbDecoder(_Handle):
    """KMC database records -> batch on one GPU (kmcb200_kmcdb_*), what `kmc -fkmc` reads: every .kmc_suf record whose counter passes the
    database's cutoffs becomes its k-mer in ACGT and one '\\n', in file order, byte for byte kmc_b200.reads.kmc_db_to_batch.  `lut` is the
    LUT as the reference's listing reader sees it (kmc_b200.reads.kmc_db_info gives it); it stays in HBM.  A chunk is whole records, of
    at most max_records; first_record is the index of its first record in the file."""
    _prefix = "kmcb200_kmcdb"

    def __init__(self, kmer_len, lut_prefix_len, counter_size, min_count, max_count, total_kmers, lut, device=0, max_records=1 << 22):
        self.kmer_len, self.lut_prefix_len, self.counter_size = int(kmer_len), int(lut_prefix_len), int(counter_size)
        self.record_bytes = (self.kmer_len - self.lut_prefix_len) // 4 + self.counter_size
        self.max_records = int(max_records)
        self.last_kept = self.last_seq_bytes = 0
        lut = np.ascontiguousarray(lut, dtype=np.uint64)
        p = _KmcDbParams(device, self.kmer_len, self.lut_prefix_len, self.counter_size, int(min_count), min(int(max_count), (1 << 64) - 1),
                         int(total_kmers), self.max_records)
        self._open(C.byref(p), lut.ctypes.data, lut.size)

    def kernel_launches(self):
        return int(self.lib.kmcb200_kmcdb_kernel_launches(self._h))

    def records_in(self, a):
        if self.record_bytes and a.size % self.record_bytes:
            raise KmcB200Error(ERR_INVALID, "%d bytes are not whole records of %d bytes" % (a.size, self.record_bytes))
        return a.size // self.record_bytes if self.record_bytes else 0

    def decode(self, suffix, first_record, out=None):
        """kmcb200_kmcdb_decode: the batch of the records (a uint8 view of `out`, default fresh n * (k + 1) bytes); a shorter `out` than
        the batch raises ERR_CAPACITY and is left untouched.  The records kept are left in last_kept."""
        a = _as_u8(suffix)
        n = self.records_in(a)
        o = np.empty(n * (self.kmer_len + 1), dtype=np.uint8) if out is None else out
        nbytes, kept = C.c_uint64(0), C.c_uint64(0)
        rc = self.lib.kmcb200_kmcdb_decode(self._h, a.ctypes.data, n, int(first_record), o.ctypes.data, o.size, C.byref(nbytes), C.byref(kept))
        self.last_seq_bytes, self.last_kept = int(nbytes.value), int(kept.value)
        self._check(rc)
        return o[:nbytes.value]

    def dev_decode(self, d_suffix, n_records, first_record, d_seq, capacity, d_result, stream=None):
        """kmcb200_dev_kmcdb_decode: device pointers (ints or tensors' data_ptr()); d_result receives 2 x uint64: sequence bytes, records
        kept (d_seq is not written when the first exceeds capacity)."""
        self._check(self.lib.kmcb200_dev_kmcdb_decode(self._h, d_suffix, int(n_records), int(first_record), d_seq, int(capacity), d_result, stream))


class Gunzip(_Handle):
    """BGZF members inflated on one GPU (kmcb200_gunzip_*): one warp per member, the text zlib's byte for byte, every member's CRC32 and
    ISIZE checked.  A malformed member raises ERR_INVALID with its offset and leaves text_out unwritten.  Plain (non-BGZF) gzip is serial:
    kmc_b200.reads inflates it with zlib."""
    _prefix = "kmcb200_gunzip"

    def __init__(self, device=0, max_in_bytes=1 << 26, max_out_bytes=1 << 26):
        self.max_in_bytes, self.max_out_bytes = max_in_bytes, max_out_bytes
        p = _GunzipParams(device, 0, max_in_bytes, max_out_bytes)
        self._open(C.byref(p))

    def kernel_launches(self):
        return int(self.lib.kmcb200_gunzip_kernel_launches(self._h))

    def inflate(self, raw, text_out):
        """kmcb200_gunzip_inflate: the whole BGZF members at the start of raw (at most max_in_bytes, ideally pinned) whose text fits
        text_out (uint8, ideally pinned) are inflated into it.  Returns (consumed, text_bytes); (0, 0) when not one whole member fits.
        ERR_INVALID when raw does not start with a BGZF member."""
        a = _as_u8(raw)
        consumed, nbytes = C.c_uint64(0), C.c_uint64(0)
        self._check(self.lib.kmcb200_gunzip_inflate(self._h, a.ctypes.data, a.size, text_out.ctypes.data, text_out.size, C.byref(consumed),
                                                    C.byref(nbytes)))
        return int(consumed.value), int(nbytes.value)

    def dev_inflate(self, d_members, n_members, d_raw, raw_bytes, d_text, text_capacity, d_error, stream=None):
        """kmcb200_dev_gunzip_inflate: device pointers (ints or tensors' data_ptr()); d_members holds a bgzf_scan table; d_error receives ~0,
        or min over the bad members of (index << 8 | error code)."""
        self._check(self.lib.kmcb200_dev_gunzip_inflate(self._h, d_members, n_members, d_raw, raw_bytes, d_text, text_capacity, d_error, stream))


def bgzf_scan(raw, capacity, max_members=None):
    """kmcb200_bgzf_scan (host only, no GPU): the whole BGZF members at the start of raw whose text fits `capacity` bytes.  Returns
    (consumed, text_bytes, members), members a BGZF_MEMBER array (in_off, out_off, in_bytes, isize).  ERR_INVALID when raw does not start
    with a BGZF member."""
    lib = load_library()
    a = _as_u8(raw)
    cap = a.size // BGZF_MIN_MEMBER + 1 if max_members is None else int(max_members)
    members = np.zeros(cap, dtype=BGZF_MEMBER)
    consumed, text, n = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    rc = lib.kmcb200_bgzf_scan(a.ctypes.data, a.size, int(capacity), members.ctypes.data, cap, C.byref(consumed), C.byref(text), C.byref(n))
    if rc < 0:
        raise KmcB200Error(rc, (lib.kmcb200_gunzip_last_error(None) or b"").decode())
    return int(consumed.value), int(text.value), members[:n.value]


def _host_check(lib, rc):
    if rc < 0:
        raise KmcB200Error(rc, (lib.kmcb200_sigstats_last_error(None) or b"").decode())


def signature_map(counts, signature_len, n_bins):
    """CSignatureMapper::Init (kmc_core/s_mapper.h:141-235) on the host: int32[4^signature_len + 1] bin ids from per-signature k-mer counts,
    -1 for the signatures that are not allowed (no k-mer has them).  Needs no GPU."""
    lib = load_library()
    cnt = np.ascontiguousarray(counts, dtype=np.uint32)
    if cnt.size != (1 << (2 * signature_len)) + 1:
        raise KmcB200Error(ERR_INVALID, "counts has %d entries, 4^%d + 1 expected" % (cnt.size, signature_len))
    out = np.zeros(cnt.size, dtype=np.int32)
    _host_check(lib, lib.kmcb200_signature_map(cnt.ctypes.data, signature_len, n_bins, out.ctypes.data))
    return out


def stage2_bin_order(bytes_per_bin, n_rec, n_plus_x_recs, kmer_len, cutoff_min, cutoff_max, counter_max, lut_prefix_len):
    """The reference's stage-2 order of the bins with one thread (CBinDesc::get_sorted_req_sizes, kmc_core/queues.h:499-558) on the host:
    uint32[n_bins], every bin's position in the database.  Needs no GPU."""
    lib = load_library()
    b = np.ascontiguousarray(bytes_per_bin, dtype=np.uint64)
    r = np.ascontiguousarray(n_rec, dtype=np.uint64)
    x = None if n_plus_x_recs is None else np.ascontiguousarray(n_plus_x_recs, dtype=np.uint64)
    if r.size != b.size or (x is not None and x.size != b.size):
        raise KmcB200Error(ERR_INVALID, "per-bin arrays of different lengths")
    out = np.zeros(b.size, dtype=np.uint32)
    _host_check(lib, lib.kmcb200_stage2_bin_order(b.size, b.ctypes.data, r.ctypes.data, None if x is None else x.ctypes.data, kmer_len, cutoff_min,
                                                  min(int(cutoff_max), (1 << 64) - 1), min(int(counter_max), (1 << 64) - 1), lut_prefix_len,
                                                  out.ctypes.data))
    return out
