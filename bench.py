#!/usr/bin/env python3
"""bench.py -- marker-scan throughput on H100 (BASELINE.json metric: YAML MB/s scanned + markers/s,
% of the HBM-read roofline, next to the reference's CPU path).

    python bench.py --gpus N --steps K --warmup W            (N>1: launched under torch.distributed.run)
    python bench.py --impl reference ...                     (the reference's CPU path on the host cores)
    python bench.py ... --dump-outputs DIR                   (also write what the last timed step computed)

A "step" is one pass of the hot path over the whole synthetic batch:
  workload  BASELINE.json configs[3] / the north-star target: 2,621,440 synthetic manifests x 4,096 B
            = 10 GiB (generator: obm_corpus.h, splitmix64(0x0B200 ^ doc index), 8 markers per file),
            resident in HBM, sharded by file over the N ranks ("strong" scaling: total work fixed).
            Inputs are 10 GiB >> 50 MB L2, so no L2 flush is needed between timed iterations.
  value     total input MB / device time of (scan + emit [+ the N>1 index all-gather]), max over ranks
  e2e       the same metric through the C-ABI host entry point obm_lex_batch: pinned host buffers,
            H2D of the manifests and D2H of tuples + offsets inside the timed region (bounded sample)
  roofline  algorithmic bytes = 1 byte read per input byte (SURVEY.md 8d) / time of all scan kernels,
            against the HBM copy peak in MEASURED_PEAKS.json if present, else the H100 SXM data sheet's 3.35 TB/s
  cpu_baseline  the oracle (C restatement of the reference's Go lexer) on all host cores over a bounded
            sample of the same corpus
  gpu       the card's name, power limit and maximum SM clock: every number above belongs to them

--dump-outputs DIR writes, after the timed steps, what the last step left for its caller as float64 .npy files: the
tuple stream of rank 0's shard (a fixed, seeded sample of its words, split into kind / off / len), the per-document tuple
offsets (sampled the same way above 2^20 documents), the marker and lexeme counts and the status words; with N > 1 also
a sample of the all-gathered marker index.  The corpus is a function of the arguments, so two builds run with the same
arguments can be compared file for file.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DOC_BYTES = 4096
FULL_DOCS = 2_621_440  # 10 GiB
FALLBACK_HBM_GBS = 3350.0  # H100 SXM data sheet, used when MEASURED_PEAKS.json is absent
DUMP_ROWS = 1 << 20  # rows per sampled array of --dump-outputs: 8 B each as float64, under 64 MB in all


def measured_peak():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return FALLBACK_HBM_GBS, "H100 SXM data sheet (3.35 TB/s), not measured"


def gpu_info(gpu_index):
    """name, power limit and maximum SM clock of the card the numbers are measured on"""
    try:
        row = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(gpu_index)], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": row[0].strip(), "power_limit_w": float(row[1]), "sm_max_mhz": float(row[2])}
    except Exception:
        return None


def sample_rows(n, k, seed):
    """sorted row indices: all n rows, or a fixed seeded sample of about k of them"""
    import numpy as np
    if n <= k:
        return np.arange(n, dtype=np.int64)
    return np.unique(np.random.default_rng(seed).integers(0, n, k, dtype=np.int64))


def dump_outputs(out_dir, d_out, n_tuples, d_toff, d_counts, d_status, index=None):
    """writes what the step left in the caller's buffers as DIR/<name>.npy (float64; a tuple word is split into its
    kind / off / len fields, include/obmarkers.h, because float64 holds only 53 bits)"""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    dev = d_out.device
    ti = sample_rows(n_tuples, DUMP_ROWS, 1)
    t = d_out[torch.from_numpy(ti).to(dev)].cpu().numpy().view(np.uint64)
    di = sample_rows(d_toff.numel(), DUMP_ROWS, 2)
    arrays = {"tuple_index": ti, "tuple_kind": t >> np.uint64(59), "tuple_len": (t >> np.uint64(32)) & np.uint64(0x7FFFFFF),
              "tuple_off": t & np.uint64(0xFFFFFFFF), "doc_index": di,
              "doc_tuple_off": d_toff[torch.from_numpy(di).to(dev)].cpu().numpy(),
              "counts": np.array([n_tuples] + d_counts.cpu().tolist()), "status": d_status.cpu().numpy()}
    if index is not None:  # N > 1: the all-gathered marker index, records {doc, tuple, off, registry id | scope count << 16}
        ii = sample_rows(index.shape[0], DUMP_ROWS // 4, 3)
        arrays["marker_index_row"] = ii
        arrays["marker_index"] = index[torch.from_numpy(ii).to(dev)].cpu().numpy().view(np.uint32)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), np.ascontiguousarray(a, dtype=np.float64))


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.gpu = gpu_index
        self.rows = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100",
                                          "-i", str(self.gpu)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx = float(f[2])
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


def host_threads():
    """threads the CPU legs may use: the affinity / cgroup view, not os.cpu_count()"""
    try:
        return max(1, len(os.sched_getaffinity(0)))
    except Exception:
        return os.cpu_count() or 1


def cpu_reference_run(sample_docs, threads, steps, warmup, flavour):
    """Times the oracle (C restatement of internal/markers/lexer) over a bounded sample on the host cores.  This leg maps
    oracle code only: the corpus comes from oracle/libcorpus_gen.so (the generator's host build), not from libobmarkers.so."""
    import oracle
    data, off = oracle.generate_corpus(sample_docs, DOC_BYTES, 0, flavour)
    for _ in range(max(warmup, 1)):
        oracle.scan_batch(data[:min(len(data), 4096 * DOC_BYTES)], off[:min(sample_docs, 4096) + 1], threads)
    times, markers, lexemes = [], 0, 0
    for _ in range(steps):
        t0 = time.perf_counter()
        nl, nm, _h = oracle.scan_batch(data, off, threads)
        times.append(time.perf_counter() - t0)
        markers, lexemes = nm, nl
    dt = sum(times) / len(times)
    # one thread over a slice of the same sample: what a core does
    one_docs = min(sample_docs, 2048)
    t0 = time.perf_counter()
    oracle.scan_batch(data[:one_docs * DOC_BYTES], off[:one_docs + 1], 1)
    one = one_docs * DOC_BYTES / (time.perf_counter() - t0) / 1e6
    return {"mb_s": len(data) / dt / 1e6, "ms_per_step": dt * 1e3, "markers_per_s": markers / dt, "lexemes": lexemes,
            "single_thread_mb_s": one, "pass_ms": [round(t * 1e3, 1) for t in times],
            "sample": f"{sample_docs} docs x {DOC_BYTES} B ({sample_docs * DOC_BYTES / 2**20:.0f} MiB) of the same generator, "
                      f"{steps} pass(es), {threads} pthreads"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--docs", type=int, default=int(os.environ.get("OBM_BENCH_DOCS", FULL_DOCS)), help="total documents (default 10 GiB worth)")
    ap.add_argument("--flavour", type=int, default=0)
    ap.add_argument("--e2e-docs", type=int, default=int(os.environ.get("OBM_BENCH_E2E_DOCS", 262144)), help="documents per rank in the e2e leg (1 GiB)")
    ap.add_argument("--cpu-docs", type=int, default=int(os.environ.get("OBM_BENCH_CPU_DOCS", 65536)), help="documents in the CPU baseline sample (256 MiB)")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--mode", type=int, default=0, help="0 auto (fast path), 1 exact path only")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write what the last timed step computed as DIR/<name>.npy (float64)")
    args = ap.parse_args()
    if args.dump_outputs and args.impl != "b200":
        ap.error("--dump-outputs writes the outputs of the GPU path (--impl b200)")
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else args.warmup

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    cores = host_threads()

    cfg_name = "configs[3]" if args.flavour == 0 else "configs[2] (workload-collection spelling: +operator-builder:collection:field)"
    config = {"workload": f"{cfg_name}: {args.docs} synthetic manifests x {DOC_BYTES} B = {args.docs * DOC_BYTES / 2**30:.2f} GiB, "
                          f"8 markers/file, sharded by file over {world} rank(s), HBM-resident",
              "docs": args.docs, "doc_bytes": DOC_BYTES, "flavour": args.flavour,
              "parallelism": f"file-shard x{world}; step = scan + emit" + (" + marker index (16 B per registered marker) + one NCCL all-gather of the index records (obm_lex_batch_sharded_device, C ABI)" if world > 1 else ""),
              "l2": "inputs (>= 1.25 GiB per rank) exceed the 50 MB L2; no flush needed"}

    if args.impl == "reference":
        # The reference's own CPU implementation of the path; Go cannot be built here, so this is the
        # oracle port of internal/markers/lexer on all host cores (kind "port").  Rank 0 only.
        if rank != 0:
            return 0
        # a step = one pass of the CPU path over a BOUNDED SAMPLE of the workload (1 GiB by default);
        # `config.workload` names the full workload, `config.sample` what a step really covers
        steps = args.steps
        ref_docs = max(args.cpu_docs, int(os.environ.get("OBM_BENCH_REF_DOCS", 262144)))
        r = cpu_reference_run(ref_docs, cores, steps, 1, args.flavour)
        config["sample"] = r["sample"]
        line = {"impl": "reference", "metric": "manifest_scan_throughput", "value": r["mb_s"], "unit": "MB/s", "n_gpus": world,
                "steps": steps, "warmup": 1, "ms_per_step": r["ms_per_step"], "higher_is_better": True,
                "scaling": "strong", "vs_baseline": None, "dtype": "u8", "data": "synthetic", "config": config,
                "markers_per_s": r["markers_per_s"],
                "cpu_baseline": {"value": r["mb_s"], "unit": "MB/s", "cores": cores, "kind": "port", "sample": r["sample"],
                                 "single_thread_mb_s": r["single_thread_mb_s"], "pass_ms": r["pass_ms"]},
                "e2e": {"value": r["mb_s"], "unit": "MB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                "gpu_launches": 0}
        print(json.dumps(line))
        return 0

    import numpy as np
    import torch
    import torch.distributed as dist
    import operator_builder_b200 as ob

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: operator-builder_b200 has no CPU fallback"}))
        return 2
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        # NCCL prints its banner / NCCL_DEBUG lines on stdout when the first communicator comes up; rank 0 must print exactly one
        # JSON line there, so stdout points at stderr until both communicators (torch's, and obm_comm_create's below) exist.
        # NCCL_DEBUG itself is left alone: the driver's rank check reads the lines from stderr.
        sys.stdout.flush()
        saved_stdout = os.dup(1)
        os.dup2(2, 1)
        dist.init_process_group("nccl", device_id=dev)

    from operator_builder_b200 import shard
    d0, d1 = shard.shard_range(args.docs, rank, world)
    ndocs = d1 - d0
    nbytes = ndocs * DOC_BYTES
    sc = ob.Scanner(local_rank)
    sc.set_mode(args.mode)
    stream = torch.cuda.current_stream()
    sp = stream.cuda_stream

    d_bytes = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    d_off = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
    sc.generate_corpus_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, DOC_BYTES, d0, args.flavour, sp)
    cap = nbytes // 16  # tuples (8 B each): 0.5 B of tuples per input byte; measured need is ~0.35
    d_out = torch.empty(cap, dtype=torch.int64, device=dev)
    d_toff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
    d_status = torch.zeros(4, dtype=torch.int32, device=dev)
    d_counts = torch.zeros(2, dtype=torch.int64, device=dev)
    # the parser on the device (SURVEY 8f-1): compact Result records, 32 B each + 16 B per argument
    reg = ob.Registry()
    max_docs = (args.docs + world - 1) // world
    res_cap, arg_cap = max_docs * 12, max_docs * 48
    d_res = torch.empty(res_cap * 32, dtype=torch.uint8, device=dev)
    d_args = torch.empty(arg_cap * 16, dtype=torch.uint8, device=dev)
    d_roff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
    d_tot = torch.zeros(2, dtype=torch.int64, device=dev)
    comm = d_idx = d_idx_all = None
    if world > 1:
        # the multi-GPU path behind the C ABI: obm_comm_* (NCCL bound inside libobmarkers.so); torch.distributed only carries
        # the 128-byte unique id from rank 0 to the others and the barriers / max-over-ranks of this harness
        idt = torch.zeros(128, dtype=torch.uint8, device=dev)
        if rank == 0:
            idt.copy_(torch.frombuffer(bytearray(ob.Comm.unique_id()), dtype=torch.uint8))
        dist.broadcast(idt, 0)
        comm = ob.Comm(sc, bytes(idt.cpu().numpy().tobytes()), rank, world)
        idx_cap = max_docs * 12
        d_idx = torch.empty(idx_cap * 16, dtype=torch.uint8, device=dev)
        d_idx_all = torch.empty(world * idx_cap * 16, dtype=torch.uint8, device=dev)
        warm = torch.zeros(1, device=dev); dist.all_reduce(warm); torch.cuda.synchronize()
        sys.stdout.flush(); os.dup2(saved_stdout, 1); os.close(saved_stdout)  # both communicators are up: stdout is ours again
    exch = {}

    def scan_only():
        sc.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, nbytes, d_out.data_ptr(), cap, d_toff.data_ptr(),
                            d_status.data_ptr(), d_counts.data_ptr(), sp)

    def parse_only():
        sc.parse_batch_device(reg, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, d0, d_out.data_ptr(), d_toff.data_ptr(), d_res.data_ptr(), res_cap,
                              d_args.data_ptr(), arg_cap, d_roff.data_ptr(), d_tot.data_ptr(), sp)

    def step():
        """one pass of the hot path over the rank's shard: scan + emit and (N > 1) the one exchange step -- the compact index of
        the registered markers, all-gathered over NVLink by NCCL, all behind the C ABI"""
        if comm is None:
            scan_only()  # N = 1: the lexer's work, what the reference arm times on the CPU; the parser is timed beside it (parts)
        else:
            per_rank, stride = comm.lex_batch_sharded_device(reg, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, nbytes, d0, d_out.data_ptr(), cap,
                                                             d_toff.data_ptr(), d_status.data_ptr(), d_counts.data_ptr(), d_idx.data_ptr(), idx_cap,
                                                             d_idx_all.data_ptr(), world * idx_cap, sp)
            exch["per_rank"], exch["stride"] = per_rank, stride

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        a.record(stream)
        for _ in range(n):
            fn()
        b.record(stream)
        barrier()
        return a.elapsed_time(b) / n

    for _ in range(args.warmup):
        step()
    barrier()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    ms = timed(step, args.steps)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        index = None
        if comm is not None:
            recs = d_idx_all.view(torch.int32).view(-1, 4)
            index = torch.cat([recs[r * exch["stride"]:r * exch["stride"] + exch["per_rank"][r]] for r in range(world)])
        dump_outputs(args.dump_outputs, d_out, int(d_toff[-1].item()), d_toff, d_counts, d_status, index)
    launches = (ob._native.lib().obm_launches_last_call(sc.handle) + (2 if world > 1 else 0)) * args.steps  # scan kernels (+ N > 1: the one-pass index = k_flat_tile_docs + k_marker_index_flat)

    # the parts, same stream, same events: scan-only time is the roofline's denominator
    ms_scan = timed(scan_only, args.steps)
    ms_parse = timed(parse_only, max(3, args.steps // 2))

    n_tuples = int(d_toff[-1].item())
    n_markers, n_lexemes = int(d_counts[0].item()), int(d_counts[1].item())
    n_results, n_args = [int(x) for x in d_tot.cpu().tolist()]
    status = d_status.cpu().tolist()
    if status[0]:
        print(json.dumps({"error": "tuple buffer overflow in bench", "needed": n_tuples, "cap": cap}))
        return 3

    # full-tuple all-gather, timed separately (SURVEY.md section 7 hard part 1: at 0.35 B/B it moves more bytes per GPU than the
    # scan reads at N=8, so the path exchanges the parser's records instead and the tuples stay resident on their owner)
    gather = None
    if world > 1:
        mx = torch.tensor([n_tuples], dtype=torch.int64, device=dev)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        pad = int(mx.item())
        g_out = torch.empty(pad * world, dtype=torch.int64, device=dev)
        src = d_out[:pad]
        gms = timed(lambda: dist.all_gather_into_tensor(g_out, src), 3)
        gather = {"ms": gms, "bytes_received_per_rank": pad * 8 * (world - 1), "gb_s_per_rank": pad * 8 * (world - 1) / gms / 1e6}
        del g_out

    # max over ranks
    t = torch.tensor([ms, ms_scan, ms_parse], dtype=torch.float64, device=dev)
    agg = torch.tensor([n_tuples, n_markers, n_lexemes, status[1], status[2], n_results, n_args], dtype=torch.int64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(agg, op=dist.ReduceOp.SUM)
    ms, ms_scan, ms_parse = [float(x) for x in t.tolist()]
    tot_tuples, tot_markers, tot_lexemes, docs_exact, docs_fatal, tot_results, tot_args = [int(x) for x in agg.tolist()]
    total_bytes = args.docs * DOC_BYTES

    # ---- e2e: C-ABI host entry point, pinned host buffers, H2D + D2H inside the timed region ----
    e2e = None
    if not args.no_e2e:
        e_docs = min(args.e2e_docs, ndocs)
        e_bytes = e_docs * DOC_BYTES
        h_bytes = torch.empty(e_bytes, dtype=torch.uint8).pin_memory()
        h_bytes.copy_(d_bytes[:e_bytes])
        h_off = np.arange(e_docs + 1, dtype=np.uint64) * DOC_BYTES
        e_cap = e_bytes // 16
        h_out = torch.empty(e_cap, dtype=torch.int64).pin_memory()
        hb, ho = h_bytes.numpy(), h_out.numpy().view(np.uint64)
        del d_out
        torch.cuda.empty_cache()
        res = sc.lex_batch(hb, h_off, out=ho)  # warm-up (allocates the handle's device staging)
        res = sc.lex_batch(hb, h_off, out=ho)
        barrier()
        t0 = time.perf_counter()
        e_steps = max(3, min(args.steps, 10))
        for _ in range(e_steps):
            res = sc.lex_batch(hb, h_off, out=ho)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / e_steps
        et = torch.tensor([dt], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(et, op=dist.ReduceOp.MAX)
        dt = float(et.item())
        d2h = int(res.stats["n_tuples"]) * 8 + (e_docs + 1) * 8
        e2e = {"value": e_bytes * world / dt / 1e6, "unit": "MB/s", "h2d_bytes_per_step": e_bytes + (e_docs + 1) * 8,
               "d2h_bytes_per_step": d2h, "ms_per_step": dt * 1e3, "api": "obm_lex_batch (C ABI, pinned host buffers)",
               "sample": f"{e_docs} docs x {DOC_BYTES} B per rank", "markers_per_s": res.stats["n_markers"] * world / dt,
               "ms_kernels_inside": res.stats["ms_kernels"]}

    if comm is not None:
        comm.close()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return 0

    peak, peak_src = measured_peak()
    achieved = (total_bytes / world) / (ms_scan / 1e3) / 1e9  # per-GPU GB/s of algorithmic input bytes
    cpu = None
    if not args.no_cpu and world >= 1:
        r = cpu_reference_run(args.cpu_docs, cores, 2, 1, args.flavour)
        cpu = {"value": r["mb_s"], "unit": "MB/s", "cores": cores, "kind": "port", "sample": r["sample"],
               "markers_per_s": r["markers_per_s"], "single_thread_mb_s": r["single_thread_mb_s"]}

    line = {"metric": "manifest_scan_throughput", "value": total_bytes / (ms / 1e3) / 1e6, "unit": "MB/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "u8", "data": "synthetic", "config": config,
            "markers_per_s": tot_markers / (ms / 1e3), "lexemes_per_s": tot_lexemes / (ms / 1e3),
            "tuples": tot_tuples, "tuple_bytes_per_input_byte": tot_tuples * 8 / total_bytes,
            "docs_exact_path": docs_exact, "docs_fatal": docs_fatal, "mode": args.mode,
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "peak_source": peak_src, "ms_scan_kernels": ms_scan,
                         "algorithmic_bytes_per_launch": total_bytes // world,
                         "note": "1 B read per input byte (SURVEY 8d); time = all kernels of one scan, per GPU"},
            "cpu_baseline": cpu, "e2e": e2e, "gpu_launches": launches, "clocks": clocks, "gpu": gpu_info(local_rank),
            "parts": {"ms_scan": ms_scan, "ms_parse": ms_parse, "results": tot_results, "args": tot_args,
                      "result_bytes_per_input_byte": tot_results * 32 / total_bytes},
            "exchange": ({"in_step": "ncclAllGather of 16-byte marker-index records (+ an 8-byte count gather), through the C ABI",
                          "records_per_rank": exch.get("per_rank"), "slot_stride": exch.get("stride"),
                          "bytes_received_per_rank": (exch.get("stride") or 0) * 16 * (world - 1),
                          "full_tuple_allgather_not_in_step": gather} if world > 1 else None)}
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
