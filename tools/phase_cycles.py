#!/usr/bin/env python3
"""Where k_warp_scan<false>'s cycles go: per-phase cycle accounting of the fused warp kernel on the bench corpus
(configs[3], 4 KiB manifests generated on the device, HBM resident; 2 GiB by default, OBM_PHASE_DOCS documents).

Needs the phase-clock build of the library (libobmarkers_phase.so, compiled with -DOBMW_PHASE_CLOCKS; __graft_entry__.build()
makes it), selected with OBM_LIB.  The counters are clock64() differences that each warp adds up in registers between
phase borders and sums into a device array at kernel end:

  stage_wait    issuing and waiting for the unit's bulk copy
  phase_a       the bitmaps: byte classes, line starts, owners (scan_range phase A)
  phase_b       owner records: line numbers, marker or plain line (phase B)
  phase_c       the marker lines' stepper (phase C)
  assembly      counts -> tuple positions inside the unit (end of scan_range)
  assemble_fin  the unit's tuples packed into shared memory for the deferred write
  write         write_fin and write_unit: tuples to global memory
  chain         waiting in chain_resolve for the unit's exclusive prefix
  other         unit hand-out, chain_publish, the next bulk copy's issue

Prints one JSON line: cycles per unit per bucket (summed over the warps' units, divided by the units), each bucket's
share, and the card's name, power limit and maximum SM clock.  The counters cost a few registers and a clock read per
border, so the absolute numbers are those of the instrumented kernel; compare builds with each other, not with bench.py."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes

import torch
import operator_builder_b200 as ob
from operator_builder_b200 import _native

BUCKETS = ["stage_wait", "phase_a", "phase_b", "phase_c", "assembly", "assemble_fin", "write", "chain", "other"]
DOC_BYTES, warmup, steps = 4096, 3, int(os.environ.get("OBM_PHASE_STEPS", 5))
ndocs = int(os.environ.get("OBM_PHASE_DOCS", 524288))  # 2 GiB


def gpu_info():
    try:
        row = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": row[0].strip(), "power_limit_w": float(row[1]), "sm_max_mhz": float(row[2])}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None}


def main():
    L = _native.lib()
    if not hasattr(L, "obm_phase_cycles"):
        raise SystemExit(f"{_native.SO_PATH} has no phase counters: select the -DOBMW_PHASE_CLOCKS build with OBM_LIB")
    L.obm_phase_cycles.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.obm_phase_cycles.restype = ctypes.c_int
    assert L.obm_phase_buckets() == len(BUCKETS)
    counters = (ctypes.c_ulonglong * (len(BUCKETS) + 1))()

    dev = torch.device("cuda:0")
    sc = ob.Scanner(0)
    st = torch.cuda.current_stream().cuda_stream
    n = ndocs * DOC_BYTES
    cap = n // 16
    d_bytes = torch.empty(n, dtype=torch.uint8, device=dev)
    d_off = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
    sc.generate_corpus_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, DOC_BYTES, 0, 0, st)
    d_out = torch.empty(cap, dtype=torch.int64, device=dev)
    d_toff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
    d_status = torch.zeros(4, dtype=torch.int32, device=dev)
    d_counts = torch.zeros(2, dtype=torch.int64, device=dev)

    def scan():
        sc.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, n, d_out.data_ptr(), cap, d_toff.data_ptr(),
                            d_status.data_ptr(), d_counts.data_ptr(), st)

    for _ in range(warmup):
        scan()
    torch.cuda.synchronize()
    assert L.obm_phase_cycles(None, 1) == 0  # reset
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        scan()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    assert L.obm_phase_cycles(counters, 0) == 0
    units = int(counters[len(BUCKETS)])
    cyc = [int(counters[i]) for i in range(len(BUCKETS))]
    total = sum(cyc)
    print(json.dumps({"workload": f"configs[3]: {ndocs} docs x {DOC_BYTES} B = {n / 2**30:.2f} GiB, HBM resident", "lib": os.path.basename(_native.SO_PATH),
                      "steps": steps, "warmup": warmup, "ms_per_step": ms, "units": units // steps,
                      "cycles_per_unit": {b: c / units for b, c in zip(BUCKETS, cyc)}, "cycles_per_unit_total": total / units,
                      "share": {b: c / total for b, c in zip(BUCKETS, cyc)}, "status": d_status.tolist(), "gpu": gpu_info()}))
    sc.close()


if __name__ == "__main__":
    main()
