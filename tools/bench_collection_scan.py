#!/usr/bin/env python3
"""C3 at full size (1,048,576 x 4 KiB, collection flavour, generated on the device, HBM resident): the collection rewrite
fused into the scan (obm_lex_collection_batch_device) against the composition it replaces (obm_rewrite_collection_markers_device
then obm_lex_batch_device over its output).  Device time by CUDA events around the C-ABI calls, 3 warm-ups and 10 steps per
measurement, the two arms measured alternately twice in one process; then every output of the two arms is compared.
Prints one JSON line, with the card's name, power limit and maximum SM clock read in the same run."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import operator_builder_b200 as ob
from operator_builder_b200 import _native

ndocs, doc_bytes, warmup, steps = int(os.environ.get("OBM_C3_DOCS", 1048576)), 4096, 3, 10


def gpu_info():
    try:
        row = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": row[0].strip(), "power_limit_w": float(row[1]), "sm_max_mhz": float(row[2])}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}


dev = torch.device("cuda:0")
sc = ob.Scanner(0)
L = _native.lib()
st = torch.cuda.current_stream().cuda_stream
n = ndocs * doc_bytes
cap = n // 16
d_bytes = torch.empty(n + 64, dtype=torch.uint8, device=dev)
d_off = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
sc.generate_corpus_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, doc_bytes, 0, 1, st)


def outputs():
    return dict(bytes=torch.zeros(n + 64, dtype=torch.uint8, device=dev), doc_off=torch.zeros(ndocs + 1, dtype=torch.int64, device=dev),
                out=torch.zeros(cap, dtype=torch.int64, device=dev), toff=torch.zeros(ndocs + 1, dtype=torch.int64, device=dev),
                status=torch.zeros(4, dtype=torch.int32, device=dev), counts=torch.zeros(2, dtype=torch.int64, device=dev))


F, C = outputs(), outputs()


def fused():
    sc.lex_collection_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, n, F["bytes"].data_ptr(), n + 64, F["doc_off"].data_ptr(),
                                   F["out"].data_ptr(), cap, F["toff"].data_ptr(), F["status"].data_ptr(), F["counts"].data_ptr(), st)


def composition():
    # the rewrite synchronises to learn the rewritten size; the scan then reads the rewritten copy
    assert L.obm_rewrite_collection_markers_device(sc.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, C["bytes"].data_ptr(), n + 64,
                                                   C["doc_off"].data_ptr(), st) == 0
    total = int(C["doc_off"][ndocs].item())
    sc.lex_batch_device(C["bytes"].data_ptr(), C["doc_off"].data_ptr(), ndocs, total, C["out"].data_ptr(), cap, C["toff"].data_ptr(),
                        C["status"].data_ptr(), C["counts"].data_ptr(), st)


def rewrite_only():
    assert L.obm_rewrite_collection_markers_device(sc.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, C["bytes"].data_ptr(), n + 64,
                                                   C["doc_off"].data_ptr(), st) == 0


def scan_only():
    total = int(C["doc_off"][ndocs].item())
    sc.lex_batch_device(C["bytes"].data_ptr(), C["doc_off"].data_ptr(), ndocs, total, C["out"].data_ptr(), cap, C["toff"].data_ptr(),
                        C["status"].data_ptr(), C["counts"].data_ptr(), st)


def timed(fn):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


runs = []
for _ in range(2):
    runs.append({"fused_ms": timed(fused), "composition_ms": timed(composition)})
parts = {"rewrite_ms": timed(rewrite_only), "scan_of_rewritten_ms": timed(scan_only)}  # where the composition's time goes
fused()
composition()
torch.cuda.synchronize()
identical = {k: bool(torch.equal(F[k], C[k])) for k in F}
fused_ms = min(r["fused_ms"] for r in runs)
comp_ms = min(r["composition_ms"] for r in runs)
print(json.dumps({"workload": f"C3: {ndocs} docs x {doc_bytes} B, collection flavour, HBM resident", "input_bytes": n,
                  "rewritten_bytes": int(F["doc_off"][ndocs].item()), "tuples": int(F["toff"][ndocs].item()), "runs": runs, **parts,
                  "fused_best_ms": fused_ms, "composition_best_ms": comp_ms, "fused_input_GBps": n / fused_ms / 1e6,
                  "composition_input_GBps": n / comp_ms / 1e6, "speedup": comp_ms / fused_ms, "outputs_identical": identical,
                  "status": F["status"].tolist(), "gpu": gpu_info(), "warmup": warmup, "steps": steps}))
sc.close()
