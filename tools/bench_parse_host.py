#!/usr/bin/env python3
"""Host batches to parser Results, two ways, on one GPU (pinned host buffers, as bench.py's e2e leg):
  lex+host parse   obm_lex_batch (every tuple comes back), then obm_parse_doc over every document on a thread pool sized to
                   the host's cores
  parse_batch      obm_parse_batch (scan + device parser; only records, offsets and the fallback documents' tuples come
                   back), then obm_parse_doc over the fallback (OBM_R_HOST) documents only
Workloads: the C2 generator at 1 GiB (262,144 x 4 KiB, bench.py's e2e size) and the production shape -- the node-comment
inputs of tests/golden/node_comments.json (Head + "\\n" + Line + "\\n" + Foot per YAML node, mostly tiny) repeated to about
1 M documents.  Names-only operator-builder registry.  Wall time of whole steps after one warm-up; the two arms' Results
are checked equal by a hash over every document's format_doc / obm_parse_doc bytes (outside the timed steps).  Prints one
JSON line with the card's name and power limit read in the same run.  Needs a CUDA device: without one it fails."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import operator_builder_b200 as ob
from operator_builder_b200 import inspect as ins

STEPS = int(os.environ.get("OBM_BENCH_STEPS", 3))
WORKERS = os.cpu_count() or 1


def gpu_info():
    try:
        row = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": row[0].strip(), "power_limit_w": float(row[1])}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None}


def pinned(n, dtype):
    return torch.empty(max(int(n), 1), dtype=dtype).pin_memory().numpy()


def node_comment_inputs(target):
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "node_comments.json")))

    def tree(d):
        return ins.Node(d["kind"], [tree(c) for c in d["content"]] if "content" in d else None, d.get("head", ""), d.get("line", ""), d.get("foot", ""))
    inputs = []
    for m in gold["manifests"]:
        inputs += ins.collect([tree(doc) for doc in m["docs"]]).inputs
    return (inputs * (target // len(inputs) + 1))[:target]


class Host:
    """obm_parse_doc over document ranges, a task per range on the pool (ctypes drops the GIL for the call)"""

    def __init__(self, reg, data, off):
        self.L, self.reg, self.base, self.off = ob._native.lib(), reg, data.ctypes.data, off

    def parse(self, docs, tuples, toff, collect=False):
        tbase = tuples.ctypes.data
        L, reg, base, off = self.L, self.reg.handle, self.base, self.off

        def task(ds):
            out, n, outs = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_uint64(), []
            for d, t0, t1 in ds:
                rc = L.obm_parse_doc(reg, base + int(off[d]), int(off[d + 1] - off[d]), tbase + 8 * t0, t1 - t0, ctypes.byref(out), ctypes.byref(n))
                assert rc >= 0
                if collect:
                    outs.append(ctypes.string_at(out, n.value))
                L.obm_free(out)
            return outs
        items = [(int(d), int(toff[i]), int(toff[i + 1])) for i, d in enumerate(docs)]
        step = max(1, len(items) // (WORKERS * 8) + 1)
        with ThreadPoolExecutor(WORKERS) as pool:
            parts = list(pool.map(task, [items[i:i + step] for i in range(0, len(items), step)]))
        return [x for p in parts for x in p]


def run_workload(name, sc, reg, data_np, off):
    ndocs = len(off) - 1
    data = pinned(len(data_np), torch.uint8); data[:len(data_np)] = data_np
    host = Host(reg, data, off)
    # capacities from one sizing call each (a caller keeps its buffers across batches)
    lx = sc.lex_batch(data, off)
    t_out = pinned(len(lx.tuples), torch.int64).view(np.uint64)
    pb = sc.parse_batch(reg, data, off)
    caps = [len(pb.results), len(pb.args), len(pb.host_tuples)]
    res = pinned(caps[0] * 32, torch.uint8).view(ob.RESULT_DT)
    args = pinned(caps[1] * 16, torch.uint8).view(ob.ARG_DT)
    htup = pinned(caps[2], torch.int64).view(np.uint64)
    roff, hoff, tot = np.zeros(ndocs + 1, np.uint64), np.zeros(ndocs + 1, np.uint64), np.zeros(3, np.uint64)
    st = ob._native.ObmStats()
    L = ob._native.lib()
    all_docs = np.arange(ndocs)

    def arm_lex():
        r = sc.lex_batch(data, off, out=t_out)
        host.parse(all_docs, r.tuples, r.doc_tuple_off)
        return r

    def arm_parse():
        rc = L.obm_parse_batch(sc.handle, reg.handle, data.ctypes.data, off.ctypes.data, ndocs, res.ctypes.data, caps[0], args.ctypes.data, caps[1],
                               roff.ctypes.data, htup.ctypes.data, caps[2], hoff.ctypes.data, tot.ctypes.data, ctypes.byref(st))
        assert rc == 0, rc
        fb = np.nonzero(hoff[1:] > hoff[:-1])[0]
        hfo = np.zeros(len(fb) + 1, np.uint64)
        hfo[1:] = np.cumsum(hoff[fb + 1] - hoff[fb])
        host.parse(fb, htup, hfo)
        return fb

    arms = {"lex_host_parse": arm_lex, "parse_batch": arm_parse}
    times = {k: [] for k in arms}
    for k in arms:
        arms[k]()  # warm-up
    for _ in range(STEPS):
        for k, f in arms.items():  # alternate the arms
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            times[k].append((time.perf_counter() - t0) * 1e3)
    r_lex = sc.lex_batch(data, off, out=t_out)
    lex_ms_kernels = r_lex.stats["ms_kernels"]
    fb = arm_parse()
    # identical Results: hash of every document's bytes, in order
    ha = hashlib.sha256()
    for b in host.parse(all_docs, r_lex.tuples, r_lex.doc_tuple_off, collect=True):
        ha.update(len(b).to_bytes(8, "little")); ha.update(b)
    pr = ob.ParseBatchResult(reg, res[:int(tot[0])], args[:int(tot[1])], roff, htup[:int(tot[2])], hoff, {})
    hb = hashlib.sha256()
    mv = memoryview(data)
    for d in range(ndocs):
        b = pr.format_doc(d, bytes(mv[int(off[d]):int(off[d + 1])]))
        hb.update(len(b).to_bytes(8, "little")); hb.update(b)
    assert ha.digest() == hb.digest(), f"{name}: the two arms' Results differ"
    return {
        "workload": name, "docs": ndocs, "bytes": int(off[-1] - off[0]), "results": int(tot[0]), "fallback_docs": int(len(fb)),
        "lex_host_parse": {"wall_ms": min(times["lex_host_parse"]), "wall_ms_all": times["lex_host_parse"], "ms_kernels": lex_ms_kernels,
                           "d2h_bytes": len(r_lex.tuples) * 8 + (ndocs + 1) * 8},
        "parse_batch": {"wall_ms": min(times["parse_batch"]), "wall_ms_all": times["parse_batch"], "ms_kernels": st.ms_kernels,
                        "d2h_bytes": int(tot[0]) * 32 + int(tot[1]) * 16 + int(tot[2]) * 8 + 2 * (ndocs + 1) * 8,
                        "launches": int(L.obm_launches_last_call(sc.handle))},
        "results_sha256": ha.hexdigest(),
    }


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_parse_host: no CUDA device (the scan and the parser run on the GPU only)")
    gpu = gpu_info()
    sc = ob.Scanner(0)
    reg = ob.Registry()
    out = []
    ndocs = int(os.environ.get("OBM_BENCH_C2_DOCS", 262144))
    data, off = ob.generate_corpus_host(ndocs, 4096, flavour=0)
    out.append(run_workload("c2_1GiB", sc, reg, data, off))
    del data, off
    inputs = node_comment_inputs(int(os.environ.get("OBM_BENCH_NODE_DOCS", 1 << 20)))
    data = np.frombuffer(b"".join(inputs) + b"\0", dtype=np.uint8)[:-1]
    off = np.zeros(len(inputs) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in inputs])
    out.append(run_workload("node_comments_1M", sc, reg, data, off))
    sc.close()
    print(json.dumps({"bench": "bench_parse_host", "gpu": gpu, "host_workers": WORKERS, "steps": STEPS, "workloads": out}))


if __name__ == "__main__":
    main()
