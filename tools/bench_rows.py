#!/usr/bin/env python3
"""Throughput of the SURVEY 8(f) "next" rows on a synthetic HBM-resident corpus (collection flavour):
marker index over the tuple stream (rank 1), collection rewrite (rank 2), manifest split (rank 4).
Prints one JSON line; device time by CUDA events, 3 warm-ups, inputs (1 GiB) larger than L2."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import operator_builder_b200 as ob
from operator_builder_b200 import _native

ndocs, doc_bytes, steps = int(os.environ.get("OBM_ROWS_DOCS", 262144)), 4096, 10
dev = torch.device("cuda:0")
sc = ob.Scanner(0)
L = _native.lib()
st = torch.cuda.current_stream().cuda_stream
n = ndocs * doc_bytes
d_bytes = torch.empty(n + 64, dtype=torch.uint8, device=dev)
d_off = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
sc.generate_corpus_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, doc_bytes, 0, 1, st)
cap = n // 16
d_out = torch.empty(cap, dtype=torch.int64, device=dev)
d_toff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
sc.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, n, d_out.data_ptr(), cap, d_toff.data_ptr(), None, None, st)
torch.cuda.synchronize()
ntup = int(d_toff[-1])
reg = ob.Registry()
d_rec = torch.empty(ndocs * 16 * 4, dtype=torch.int32, device=dev)
d_roff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
d_rw = torch.empty(n + 64, dtype=torch.uint8, device=dev)
d_noff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)


def timed(fn):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


ms_idx = timed(lambda: L.obm_marker_index_device(sc.handle, reg.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, d_out.data_ptr(), d_toff.data_ptr(),
                                                  d_rec.data_ptr(), ndocs * 16, d_roff.data_ptr(), st))
nrec = int(d_roff[-1])
d_flat = torch.empty(ndocs * 16 * 2, dtype=torch.int64, device=dev)
d_tot = torch.zeros(4, dtype=torch.int64, device=dev)
ms_flat = timed(lambda: L.obm_marker_index_flat_device(sc.handle, reg.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, 0, d_out.data_ptr(), d_toff.data_ptr(),
                                                       ntup, d_flat.data_ptr(), ndocs * 16, d_tot.data_ptr(), st))
nflat = int(d_tot[0])
d_res = torch.empty(ndocs * 16 * 4, dtype=torch.int64, device=dev)   # 32 B per result
d_arg = torch.empty(ndocs * 48 * 2, dtype=torch.int64, device=dev)   # 16 B per argument
d_dro = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
ms_parse = timed(lambda: sc.parse_batch_device(reg, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, 0, d_out.data_ptr(), d_toff.data_ptr(), d_res.data_ptr(), ndocs * 16,
                                               d_arg.data_ptr(), ndocs * 48, d_dro.data_ptr(), d_tot.data_ptr(), st))
nres, narg = int(d_tot[0]), int(d_tot[1])
d_hash = torch.empty(ndocs, dtype=torch.int64, device=dev)
d_nh = torch.zeros(2, dtype=torch.int32, device=dev)
ms_hash = timed(lambda: L.obm_hash_batch_device(sc.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, d_out.data_ptr(), d_toff.data_ptr(), d_hash.data_ptr(), d_nh.data_ptr(), st))
ms_rw = timed(lambda: L.obm_rewrite_collection_markers_device(sc.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, d_rw.data_ptr(), n + 64, d_noff.data_ptr(), st))
ms_sp = timed(lambda: L.obm_split_docs_device(sc.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, d_rec.data_ptr(), ndocs * 16, d_roff.data_ptr(), st))
peak = 3350.0  # H100 SXM data sheet, unless MEASURED_PEAKS.json gives a measured copy peak
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass
print(json.dumps({
    "corpus": f"{ndocs} docs x {doc_bytes} B, collection flavour, HBM resident", "peak_gbs": peak,
    "marker_index": {"ms": ms_idx, "tuple_GBps": ntup * 8 / ms_idx / 1e6, "records": nrec, "record_bytes_per_input_byte": nrec * 16 / n,
                     "frac_of_peak_on_tuple_bytes": ntup * 8 / ms_idx / 1e6 / peak},
    "marker_index_flat": {"ms": ms_flat, "tuple_GBps": ntup * 8 / ms_flat / 1e6, "records": nflat},
    "device_parser": {"ms": ms_parse, "tuple_GBps": ntup * 8 / ms_parse / 1e6, "results": nres, "args": narg, "record_bytes_per_input_byte": (nres * 32 + narg * 16) / n},
    "document_hash": {"ms": ms_hash, "tuple_GBps": ntup * 8 / ms_hash / 1e6},
    "collection_rewrite": {"ms": ms_rw, "input_GBps": n / ms_rw / 1e6, "frac_of_peak": n / ms_rw / 1e6 / peak, "out_bytes": int(d_noff[-1])},
    "manifest_split": {"ms": ms_sp, "input_GBps": n / ms_sp / 1e6, "frac_of_peak": n / ms_sp / 1e6 / peak, "manifests": int(d_roff[-1])}}))
