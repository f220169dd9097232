"""ctypes binding of libobmarkers.so (include/obmarkers.h).  Fails loudly when the CUDA extension
is missing: there is no Python or CPU implementation of the scan behind it."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("OBM_LIB") or os.path.join(_HERE, "libobmarkers.so")  # OBM_LIB: a build variant (tuning experiments)

OBM_OK, OBM_E_NO_DEVICE, OBM_E_CUDA, OBM_E_CAPACITY, OBM_E_ARG, OBM_E_NOMEM = 0, -1, -2, -3, -4, -5

# every symbol include/obmarkers.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "obm_abi_version", "obm_create", "obm_destroy", "obm_last_error", "obm_lex_batch", "obm_lex_batch_device",
    "obm_scratch_bytes", "obm_generate_corpus_device", "obm_generate_corpus_host", "obm_set_mode", "obm_pinned_alloc", "obm_launches_last_call", "obm_set_chunk_bytes",
    "obm_pinned_free", "obm_stream_new", "obm_stream_next", "obm_stream_free", "obm_decode_doc", "obm_free", "obm_registry_new", "obm_registry_operator_builder", "obm_registry_add",
    "obm_comm_unique_id", "obm_comm_create", "obm_comm_destroy", "obm_lex_batch_sharded_device",
    "obm_registry_free", "obm_registry_define", "obm_parse_doc", "obm_hash_batch_device", "obm_parse_batch_device", "obm_results_format_doc", "obm_marker_index_device",
    "obm_marker_index_flat_device", "obm_rewrite_collection_markers_device", "obm_split_docs_device", "obm_lex_collection_batch_device",
    "obm_parse_batch",
]


class ObmStats(ctypes.Structure):
    _fields_ = [("n_tuples", ctypes.c_uint64), ("n_markers", ctypes.c_uint64), ("n_lexemes", ctypes.c_uint64),
                ("n_docs_exact", ctypes.c_uint64), ("n_docs_fatal", ctypes.c_uint64), ("bytes", ctypes.c_uint64),
                ("ms_kernels", ctypes.c_float), ("ms_total", ctypes.c_float)]


class ObmLexeme(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int32), ("value", ctypes.POINTER(ctypes.c_uint8)), ("value_len", ctypes.c_uint64),
                ("line", ctypes.c_int64), ("column", ctypes.c_int64)]


class NativeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libobmarkers error {code}: {msg}")
        self.code = code


_LIB = None


def lib():
    """Load libobmarkers.so (built in-tree by __graft_entry__.build() / csrc/Makefile)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(SO_PATH):
        raise ImportError(f"{SO_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a). operator-builder_b200 has no CPU fallback.")
    L = ctypes.CDLL(SO_PATH)
    vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
    L.obm_abi_version.restype = ctypes.c_int
    L.obm_create.argtypes = [ctypes.c_int, ctypes.POINTER(vp)]
    L.obm_destroy.argtypes = [vp]
    L.obm_last_error.argtypes = [vp]
    L.obm_last_error.restype = ctypes.c_char_p
    L.obm_lex_batch.argtypes = [vp, vp, vp, u32, vp, u64, ctypes.POINTER(u64), vp, ctypes.POINTER(ObmStats)]
    L.obm_lex_batch_device.argtypes = [vp, vp, vp, u32, u64, vp, u64, vp, vp, vp, vp]
    L.obm_scratch_bytes.argtypes = [u32, u64]
    L.obm_scratch_bytes.restype = u64
    L.obm_generate_corpus_device.argtypes = [vp, vp, vp, u32, u32, u64, ctypes.c_int, vp]
    L.obm_generate_corpus_host.argtypes = [vp, vp, u32, u32, u64, ctypes.c_int]
    L.obm_set_mode.argtypes = [vp, ctypes.c_int]
    L.obm_launches_last_call.argtypes = [vp]
    L.obm_launches_last_call.restype = u32
    L.obm_set_chunk_bytes.argtypes = [vp, u64]
    L.obm_set_chunk_bytes.restype = u64
    L.obm_pinned_alloc.argtypes = [u64]
    L.obm_pinned_alloc.restype = vp
    L.obm_pinned_free.argtypes = [vp]
    L.obm_stream_new.argtypes = [vp, u64, vp, u64]
    L.obm_stream_new.restype = vp
    L.obm_stream_next.argtypes = [vp, ctypes.POINTER(ObmLexeme)]
    L.obm_stream_free.argtypes = [vp]
    L.obm_decode_doc.argtypes = [vp, u64, vp, u64, ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8)), ctypes.POINTER(u64)]
    L.obm_decode_doc.restype = ctypes.c_int64
    L.obm_free.argtypes = [vp]
    L.obm_registry_new.restype = vp
    L.obm_registry_operator_builder.restype = vp
    L.obm_registry_add.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(ctypes.c_char_p), u32]
    L.obm_registry_free.argtypes = [vp]
    L.obm_registry_define.argtypes = [vp, ctypes.c_int]
    L.obm_parse_doc.argtypes = [vp, vp, u64, vp, u64, ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8)), ctypes.POINTER(u64)]
    L.obm_parse_doc.restype = ctypes.c_int64
    L.obm_rewrite_collection_markers_device.argtypes = [vp, vp, vp, u32, vp, u64, vp, vp]
    L.obm_split_docs_device.argtypes = [vp, vp, vp, u32, vp, u64, vp, vp]
    L.obm_lex_collection_batch_device.argtypes = [vp, vp, vp, u32, u64, vp, u64, vp, vp, u64, vp, vp, vp, vp]
    L.obm_marker_index_device.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, u64, vp, vp]
    L.obm_parse_batch_device.argtypes = [vp, vp, vp, vp, u32, u32, vp, vp, vp, u64, vp, u64, vp, vp, vp]
    L.obm_parse_batch.argtypes = [vp, vp, vp, vp, u32, vp, u64, vp, u64, vp, vp, u64, vp, vp, ctypes.POINTER(ObmStats)]
    L.obm_results_format_doc.argtypes = [vp, ctypes.c_char_p, u64, vp, u64, vp, u64, vp, ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8)),
                                         ctypes.POINTER(u64)]
    L.obm_results_format_doc.restype = ctypes.c_int64
    L.obm_hash_batch_device.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp]
    L.obm_comm_unique_id.argtypes = [vp]
    L.obm_comm_create.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp)]
    L.obm_comm_destroy.argtypes = [vp]
    L.obm_lex_batch_sharded_device.argtypes = [vp, vp, vp, vp, u32, u64, u32, vp, u64, vp, vp, vp, vp, u64, vp, u64,
                                               ctypes.POINTER(u64), ctypes.POINTER(u64), vp]
    L.obm_marker_index_flat_device.argtypes = [vp, vp, vp, vp, u32, u32, vp, vp, u64, vp, u64, vp, vp]
    _LIB = L
    return L
