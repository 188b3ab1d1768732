"""ctypes binding of libfiltlong_b200.so (include/filtlong_b200.h).

This is the only way Python reaches the hot path: every call lands in the hand-written sm_90a
CUDA library through its C ABI. There is no CPU or PyTorch fallback -- if the shared object is
missing, or no CUDA device is usable, the error is raised to the caller.
"""
import ctypes as C
import os

import numpy as np

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "libfiltlong_b200.so")

FL_ALIGN_BASES = 64


class FLError(RuntimeError):
    pass


class Params(C.Structure):
    _fields_ = [
        ("window_size", C.c_int32),
        ("trim", C.c_int32), ("split_set", C.c_int32), ("split", C.c_int32),
        ("min_length_set", C.c_int32), ("min_length", C.c_int32),
        ("max_length_set", C.c_int32), ("max_length", C.c_int32),
        ("min_mean_q_set", C.c_int32), ("min_window_q_set", C.c_int32),
        ("min_mean_q", C.c_double), ("min_window_q", C.c_double),
        ("length_weight", C.c_double), ("mean_q_weight", C.c_double), ("window_q_weight", C.c_double),
        ("target_bases_set", C.c_int32), ("keep_percent_set", C.c_int32),
        ("target_bases", C.c_int64),
        ("keep_percent", C.c_double),
    ]


def make_params(window_size=250, trim=False, split=None, min_length=None, max_length=None,
                min_mean_q=None, min_window_q=None, length_weight=1.0, mean_q_weight=1.0,
                window_q_weight=1.0, target_bases=None, keep_percent=None):
    """Same keyword surface as the reference CLI options (src/arguments.cpp:152-222)."""
    p = Params()
    p.window_size = window_size
    p.trim = int(bool(trim))
    p.split_set = int(split is not None)
    p.split = split or 0
    p.min_length_set = int(min_length is not None)
    p.min_length = min_length or 0
    p.max_length_set = int(max_length is not None)
    p.max_length = max_length or 0
    p.min_mean_q_set = int(min_mean_q is not None)
    p.min_mean_q = min_mean_q or 0.0
    p.min_window_q_set = int(min_window_q is not None)
    p.min_window_q = min_window_q or 0.0
    p.length_weight, p.mean_q_weight, p.window_q_weight = length_weight, mean_q_weight, window_q_weight
    p.target_bases_set = int(target_bases is not None)
    p.target_bases = target_bases or 0
    p.keep_percent_set = int(keep_percent is not None)
    p.keep_percent = keep_percent or 0.0
    return p


class Batch(C.Structure):
    _fields_ = [
        ("n", C.c_uint32), ("reserved", C.c_uint32), ("padded_bases", C.c_uint64),
        ("off", C.c_void_p), ("len", C.c_void_p), ("seq2b", C.c_void_p), ("qual", C.c_void_p),
        ("nmask", C.c_void_p), ("ascii", C.c_void_p),
    ]


class TextRecords(C.Structure):
    _fields_ = [("cap", C.c_uint64), ("name_off", C.c_void_p), ("name_len", C.c_void_p), ("comment_len", C.c_void_p),
                ("seq_off", C.c_void_p), ("qual_off", C.c_void_p), ("len", C.c_void_p), ("name_hash", C.c_void_p)]


class Summary(C.Structure):
    _fields_ = [
        ("min_q", C.c_double), ("max_q", C.c_double), ("mean_q", C.c_double), ("stdev_q", C.c_double),
        ("min_z", C.c_double), ("max_z", C.c_double),
        ("status", C.c_int32), ("reserved", C.c_int32),
        ("target", C.c_int64), ("passed_bases", C.c_int64), ("keeping", C.c_int64),
        ("total_bases", C.c_int64), ("rows_bases", C.c_int64),
    ]


class ReadResults(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("length", "mean_q", "window_q", "length_score", "passed",
                                           "first_base_in_kmer", "last_base_in_kmer", "n_bad", "n_child",
                                           "row_start")]


class RowResults(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("parent", "start", "end", "mean_q", "window_q", "length_score",
                                           "norm_mean", "norm_window", "final_score", "passed", "passed_final")]


class SynthReads(C.Structure):
    _fields_ = [
        ("n", C.c_uint32), ("flags", C.c_uint32), ("genome_bases", C.c_uint64),
        ("off", C.c_void_p), ("len", C.c_void_p), ("start", C.c_void_p), ("strand", C.c_void_p),
        ("err_ppm", C.c_void_p), ("junk_pos", C.c_void_p), ("junk_len", C.c_void_p),
        ("adap5", C.c_void_p), ("adap3", C.c_void_p),
    ]


SYNTH_INDELS = 1


# every symbol include/filtlong_b200.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("fl_ctx_create", C.c_int, [C.POINTER(Params), C.c_int, C.POINTER(_P)]),
    ("fl_device_warmup", C.c_int, [C.c_int]),
    ("fl_ctx_destroy", None, [_P]),
    ("fl_last_error", C.c_char_p, [_P]),
    ("fl_ctx_set_stream", C.c_int, [_P, _P]),
    ("fl_ctx_sync", C.c_int, [_P]),
    ("fl_ctx_set_params", C.c_int, [_P, C.POINTER(Params)]),
    ("fl_ctx_launch_count", C.c_uint64, [_P]),
    ("fl_ctx_enable_timing", C.c_int, [_P, C.c_int]),
    ("fl_ctx_reset_timing", C.c_int, [_P]),
    ("fl_ctx_kernel_time", C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    ("fl_padded_len", C.c_uint64, [C.c_int64]),
    ("fl_anchor_slot_host", None, [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    ("fl_pack_sequence", None, [C.c_char_p, C.c_char_p, C.c_int64, C.c_uint64, _P, _P, _P]),
    ("fl_kmers_add_batch", C.c_int, [_P, C.POINTER(Batch), C.c_int]),
    ("fl_kmers_add_batch_device", C.c_int, [_P, C.POINTER(Batch), C.c_int]),
    ("fl_kmers_finalize", C.c_int, [_P, C.POINTER(C.c_uint64)]),
    ("fl_kmers_contains", C.c_int, [_P, _P, C.c_uint32, _P]),
    ("fl_kmers_export", C.c_int, [_P, _P, C.c_uint64, C.POINTER(C.c_uint64)]),
    ("fl_kmers_bitmap_dev", C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_uint64)]),
    ("fl_kmers_bitmap_changed", C.c_int, [_P]),
    ("fl_kmers_release_build_state", C.c_int, [_P]),
    ("fl_kmers_probe_info", C.c_int, [_P, C.POINTER(C.c_int32)]),
    ("fl_reads_push", C.c_int, [_P, C.POINTER(Batch)]),
    ("fl_reads_push_text", C.c_int, [_P, _P, C.c_uint64, C.c_int, C.c_int, C.POINTER(TextRecords), C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    ("fl_kmers_add_text", C.c_int, [_P, _P, C.c_uint64, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                    C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    ("fl_host_alloc", C.c_int, [C.c_uint64, C.POINTER(_P)]),
    ("fl_host_free", None, [_P]),
    ("fl_host_register", C.c_int, [_P, C.c_uint64]),
    ("fl_host_unregister", None, [_P]),
    ("fl_reads_push_device", C.c_int, [_P, C.POINTER(Batch)]),
    ("fl_reads_reset", C.c_int, [_P]),
    ("fl_reads_count", C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]),
    ("fl_finalize", C.c_int, [_P, C.c_int64, C.POINTER(Summary)]),
    ("fl_norm_partial1", C.c_int, [_P, _P, _P, _P]),
    ("fl_norm_partial2", C.c_int, [_P, _P, _P, _P, _P]),
    ("fl_norm_apply", C.c_int, [_P, _P, _P, _P, _P]),
    ("fl_select_begin", C.c_int, [_P, C.c_int64, _P]),
    ("fl_select_hist", C.c_int, [_P, C.c_int, _P]),
    ("fl_select_pick", C.c_int, [_P, C.c_int, _P]),
    ("fl_select_tie_local", C.c_int, [_P, _P, C.c_int, C.c_int]),
    ("fl_select_apply", C.c_int, [_P, _P, C.c_int, _P]),
    ("fl_select_summary", C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int64, C.POINTER(Summary)]),
    ("fl_results_reads", C.c_int, [_P, C.POINTER(ReadResults)]),
    ("fl_results_rows", C.c_int, [_P, C.POINTER(RowResults)]),
    ("fl_results_pass_dev", C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_uint64)]),
    ("fl_results_pass", C.c_int, [_P, _P, C.c_uint64, C.POINTER(C.c_uint64)]),
    ("fl_comm_unique_id", C.c_int, [_P]),
    ("fl_comm_init", C.c_int, [_P, _P, C.c_int, C.c_int]),
    ("fl_comm_destroy", C.c_int, [_P]),
    ("fl_comm_info", C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("fl_kmers_broadcast", C.c_int, [_P, C.c_int]),
    ("fl_comm_allreduce_i64_host", C.c_int, [_P, _P, C.c_int]),
    ("fl_comm_collective_count", C.c_uint64, [_P]),
    ("fl_synth_qual_device", C.c_int, [_P, C.c_uint64, C.c_uint32, _P, _P, _P, C.c_uint64, _P]),
    ("fl_synth_qual_host", None, [C.c_uint64, C.c_uint32, _P, _P, _P, C.c_uint64, _P]),
    ("fl_synth_genome_device", C.c_int, [_P, C.c_uint64, C.c_uint64, _P]),
    ("fl_synth_genome_host", None, [C.c_uint64, C.c_uint64, _P]),
    ("fl_synth_reads_device", C.c_int, [_P, C.c_uint64, _P, C.POINTER(SynthReads), C.c_uint64, _P]),
    ("fl_synth_reads_host", None, [C.c_uint64, _P, C.POINTER(SynthReads), C.c_uint64, _P]),
    ("fl_synth_assembly_device", C.c_int, [_P, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32, _P, _P]),
    ("fl_synth_assembly_host", None, [C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32, _P, _P]),
    ("fl_synth_ascii_device", C.c_int, [_P, C.c_uint32, _P, _P, _P, _P, _P]),
    ("fl_synth_ascii_host", None, [C.c_uint32, _P, _P, _P, _P, _P]),
    ("fl_version", C.c_char_p, []),
    ("fl_phred_luts", None, [C.c_int32, _P, _P]),
]

_lib = None


def lib():
    """Loads the CUDA library. Raises FLError if it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FLError("%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(filtlong_b200 has no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


SYNTH_LIB_PATH = os.path.join(PKG, "libflsynth_host.so")
_synth = None


def synth_host_lib():
    """The host-only synthetic generators (libflsynth_host.so, no CUDA inside): what the CPU legs of
    bench.py use to write their sample files, so that they never map the CUDA library."""
    global _synth
    if _synth is None:
        L = C.CDLL(SYNTH_LIB_PATH)
        for name, res, args in SYMBOLS:
            if name.startswith("fl_synth_") and name.endswith("_host"):
                fn = getattr(L, name)
                fn.restype = res
                fn.argtypes = args
        _synth = L
    return _synth


def check(ctx_handle, rc, what):
    if rc != 0:
        msg = lib().fl_last_error(ctx_handle)
        raise FLError("%s failed (%d): %s" % (what, rc, msg.decode() if msg else ""))


def ptr(a):
    """Host pointer of a numpy array / device pointer of a torch tensor / None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return int(a)
