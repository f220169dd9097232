#!/usr/bin/env python3
"""C4 at full size (2,621,440 x 4 KiB, standalone markers, generated and lexed on the device, HBM resident): the device parser
(obm_parse_batch_device) with the names-only operator-builder registry (Registry(), what bench.py's parts.ms_parse times)
against the typed one (Registry.define(FIELD, COLLECTION, RESOURCE): k_parse_docs<., true>, SetArgument / InflateObject).
Device time by CUDA events around the C-ABI call, 3 warm-ups and 10 steps per measurement, the two arms measured alternately
three times in one process; then the two arms' records are compared (the generator writes only well-typed markers, so they
must be equal).  Prints one JSON line, with the card's name, power limit and maximum SM clock read in the same run.
Needs a CUDA device: without one it fails."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import operator_builder_b200 as ob

ndocs, doc_bytes, warmup, steps = int(os.environ.get("OBM_C4_DOCS", 2621440)), 4096, 3, 10


def gpu_info():
    try:
        row = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": row[0].strip(), "power_limit_w": float(row[1]), "sm_max_mhz": float(row[2])}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}


if not torch.cuda.is_available():
    raise SystemExit("bench_parse_typed: no CUDA device (the parser runs on the GPU only)")
dev = torch.device("cuda:0")
sc = ob.Scanner(0)
st = torch.cuda.current_stream().cuda_stream
n = ndocs * doc_bytes
cap = n // 16
d_bytes = torch.empty(n, dtype=torch.uint8, device=dev)
d_off = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
sc.generate_corpus_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, doc_bytes, 0, 0, st)
d_tup = torch.empty(cap, dtype=torch.int64, device=dev)
d_toff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
d_status = torch.zeros(4, dtype=torch.int32, device=dev)
sc.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, n, d_tup.data_ptr(), cap, d_toff.data_ptr(), d_status.data_ptr(), None, st)
torch.cuda.synchronize()
assert int(d_status[0].item()) == 0 and int(d_status[3].item()) == 0
res_cap, arg_cap = ndocs * 12, ndocs * 48  # as bench.py sizes them


def outputs():
    return dict(res=torch.zeros(res_cap * 32, dtype=torch.uint8, device=dev), args=torch.zeros(arg_cap * 16, dtype=torch.uint8, device=dev),
                roff=torch.zeros(ndocs + 1, dtype=torch.int64, device=dev), tot=torch.zeros(2, dtype=torch.int64, device=dev))


arms = {"untyped": (ob.Registry(), outputs()),
        "typed": (ob.Registry.define(ob.FIELD_MARKER, ob.COLLECTION_MARKER, ob.RESOURCE_MARKER), outputs())}


def run(name):
    reg, o = arms[name]
    sc.parse_batch_device(reg, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, 0, d_tup.data_ptr(), d_toff.data_ptr(), o["res"].data_ptr(), res_cap,
                          o["args"].data_ptr(), arg_cap, o["roff"].data_ptr(), o["tot"].data_ptr(), st)


def timed(name):
    for _ in range(warmup):
        run(name)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        run(name)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


ms = {"untyped": [], "typed": []}
for _ in range(3):
    for name in ("untyped", "typed"):
        ms[name].append(round(timed(name), 4))
U, T = arms["untyped"][1], arms["typed"][1]
nres, nargs = [int(x) for x in U["tot"].tolist()]
equal = (torch.equal(U["tot"], T["tot"]) and torch.equal(U["roff"], T["roff"]) and torch.equal(U["res"][:nres * 32], T["res"][:nres * 32])
         and torch.equal(U["args"][:nargs * 16], T["args"][:nargs * 16]))
best_u, best_t = min(ms["untyped"]), min(ms["typed"])
print(json.dumps({"tool": "bench_parse_typed", "gpu": gpu_info(), "corpus": {"config": "C4", "docs": ndocs, "doc_bytes": doc_bytes, "flavour": 0},
                  "warmup": warmup, "steps": steps, "ms_untyped": ms["untyped"], "ms_typed": ms["typed"],
                  "typed_over_untyped": round(best_t / best_u, 4), "results": nres, "args": nargs, "records_equal": bool(equal)}))
sc.close()
sys.exit(0 if equal else 1)
