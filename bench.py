#!/usr/bin/env python3
"""bench.py -- registrations/sec on synthetic 64-ring scan pairs (BASELINE.json metric).

  python bench.py --gpus N --steps K --warmup W            # our CUDA path (one rank per GPU under torchrun)
  python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle restatement) on host cores
  python bench.py --scene dense ...                        # the back end at BASELINE's correspondence count (L ~ 3 k)

A "step" is one pass of the whole hot path (voxel -> FPFH -> match -> TIM graph -> max clique ->
GNC-TLS + COTE) over one batch of `--pairs` synthetic 64-ring pairs per GPU (BASELINE configs[2]: 256
pairs on 1 GPU; 8 ranks x 256 = configs[3]'s 2048 pairs).  Pairs are independent, so ranks shard them
(weak scaling) and the only collective is one NCCL all_gather of the fixed-size result records.

Workloads (`--scene`):
  street  config/params.yaml defaults on the street scene: ~111 k returns -> ~6.9 k voxel points -> ~1.8 k mutual
          nearest neighbours -> ~300 correspondences after the tuple test (the default; the headline line).
  dense   the same scans with voxel 0.22 m and the tuple test off (qb200_params.use_tuple_test = 0): ~10 k voxel points and
          L ~ 3 k correspondences per pair, the size BASELINE.json quotes for the back end (K8 graph, K9 clique, K10 pose).
          The default run measures it too, as the `dense` object of the one JSON line.

  value : whole-job registrations/s with the raw scans already resident in HBM (device pointers through
          qb200_register_batch), CUDA events on the launching stream, max over ranks.
  e2e   : the same call with pinned HOST buffers -- H2D of every scan and D2H of the result records are
          inside the timed region.
  roofline      : the dominant kernel (tc_nn_kernel, the N_src x N_tgt x 33 contraction on wgmma) from CUDA events
                  recorded around it inside the timed steps.
  cpu_baseline  : the CPU oracle (restatement of the reference path; the reference binary itself needs
                  PCL/FLANN/pmc) timed on the host's cores on a bounded sample of the same pairs.

  --dump-outputs DIR : after the timed steps, the result records of the last step (what qb200_register_batch hands
                  its caller) as DIR/<field>.npy in float64, one array per record field, all finite (the +inf `cost` of a
                  pair whose GNC stopped before evaluating one is split into cost.npy and cost_evaluated.npy).  The inputs are seeded, so two
                  builds run with the same arguments can be compared output for output.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

METRIC = "registrations/sec (64-ring pair)"
UNIT = "registrations/s"

SCENES = {
    "street": {"params": {}, "cfg": {},
               "what": "config/params.yaml defaults (voxel 0.3, normal_r 0.5, fpfh_r 0.75, noise_bound 0.3, PMC_HEU, median COTE)"},
    "dense": {"params": {"voxel_size": 0.22, "use_tuple_test": 0}, "cfg": {"max_corr": 8192},
              "what": "voxel 0.22 m, tuple test off (every mutual nearest neighbour is a correspondence): L ~ 3 k per pair; "
                      "other parameters = config/params.yaml"},
    # BASELINE configs[4]: dense indoor pair, ~500 k points, 0.05 m voxel -- the configuration where K6 (N_src x N_tgt x 33 on the
    # tensor cores) is the dominant work (34-53 k voxel points per cloud: 66 * 45k^2 = 0.13 TFLOP per pair)
    "indoor": {"params": {"voxel_size": 0.05, "normal_radius": 0.10, "fpfh_radius": 0.15, "noise_bound": 0.05, "cote_noise_bound": 0.05,
                          "skip_flagged": 0},
               "cfg": {"max_raw_points": 524288, "max_voxel_points": 65536},
               "what": "voxel 0.05 m, normal_r 0.10, fpfh_r 0.15, noise_bound 0.05 (the reference's ratios of config/params.yaml:17-25 scaled to "
                       "the voxel), floor kept (no ground removal indoors)"},
}


def scene_params(scene):
    from quatro_b200.capi import default_params
    p = default_params()
    for k, v in SCENES[scene]["params"].items():
        setattr(p, k, v)
    return p


def _host_threads() -> int:
    """Threads for the CPU arm: usable cores (affinity, cgroup quota), one per physical core (SMT siblings only
    oversubscribe the OpenMP loops)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:
        quota, period = Path("/sys/fs/cgroup/cpu.max").read_text().split()
        if quota != "max":
            n = min(n, max(1, int(quota) // int(period)))
    except (OSError, ValueError):
        pass
    try:
        sib = Path("/sys/devices/system/cpu/cpu0/topology/thread_siblings_list").read_text().strip()
        smt = len(sib.replace("-", ",").split(",")) if sib else 1
        if "-" in sib:
            a, b = sib.split("-")[:2]
            smt = int(b) - int(a) + 1
        if smt > 1 and n >= (os.cpu_count() or n):
            n = max(1, n // smt)
    except (OSError, ValueError):
        pass
    return n


def load_peaks():
    f = ROOT / "MEASURED_PEAKS.json"
    if f.exists():
        d = json.loads(f.read_text())
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"], "bf16_tflops_sustained": d.get("bf16_tflops_sustained"),
                "source": "measured (MEASURED_PEAKS.json)"}
    # NVIDIA H100 SXM data sheet (dense, 700 W card): denominators only, never reached figures
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": None, "source": "H100 SXM data sheet (not measured)"}


def dump_outputs(path, records):
    """The result records of the last timed step, one float64 array per field (T: P x 16, column-major 4 x 4 poses).
    `cost` is +inf where GNC stops before its first cost evaluation (every residual already inside the noise bound, as
    Quatro::cost_ does); it is written as cost.npy (0 there) and cost_evaluated.npy (1 where a cost was evaluated)."""
    d = Path(path)
    d.mkdir(parents=True, exist_ok=True)
    for name in records.dtype.names:
        v = records[name].astype(np.float64)
        if name == "cost":
            ok = np.isfinite(v)
            np.save(d / "cost_evaluated.npy", ok.astype(np.float64))
            v = np.where(ok, v, 0.0)
        np.save(d / f"{name}.npy", v)


def gen_pairs(seeds, scene="street"):
    from quatro_b200 import synth
    synth._lib()  # build/load once before the threads start
    make = (lambda s: synth.indoor_pair(int(s))[:2]) if scene == "indoor" else (lambda s: synth.outdoor_pair(int(s))[:2])
    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 8)) as ex:
        return list(ex.map(make, seeds))


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, device):
        self.device, self.proc, self.lines = device, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100", "-i", str(self.device)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for ln in self.proc.stdout:
            self.lines.append(ln.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": float(max(mx)) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def cpu_pair_parallel(pairs, p, cores, seconds):
    """Best-case CPU line (SURVEY.md 8d): `cores` pairs in flight, one single-threaded oracle call each (the reference itself is
    not re-entrant, so this is what one process per core would reach).  Returns (registrations/s, pairs done)."""
    from oracle import Oracle
    o = Oracle()
    done = [0] * cores
    stop_at = time.perf_counter() + seconds

    def work(k):
        o.set_num_threads(1)  # OpenMP ICV of this host thread
        i = k
        while time.perf_counter() < stop_at:
            s, t = pairs[i % len(pairs)]
            o.register_pair(s, t, p)
            done[k] += 1
            i += cores

    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=cores) as ex:
        list(ex.map(work, range(cores)))
    dt = time.perf_counter() - t0
    return sum(done) / dt, sum(done)


def run_reference(args, rank, world):
    """The reference's CPU path (oracle restatement) on the host cores; rank 0 only."""
    if rank != 0:
        return
    from oracle import Oracle
    o = Oracle()
    cores = o.set_num_threads(_host_threads())   # torchrun exports OMP_NUM_THREADS=1: ask for every usable host core explicitly
    p = scene_params(args.scene)
    per_step = args.ref_pairs_per_step
    pairs = gen_pairs(range(per_step), args.scene)
    for _ in range(max(args.warmup, 1)):
        o.register_pair(pairs[0][0], pairs[0][1], p)
    t0 = time.perf_counter()
    done = 0
    for _ in range(args.steps):
        for s, t in pairs:
            o.register_pair(s, t, p)
            done += 1
    dt = time.perf_counter() - t0
    val = done / dt
    best, best_n = cpu_pair_parallel(pairs, p, cores, min(10.0, max(3.0, dt)))
    sample = (f"{per_step} of the workload's pairs per step x {args.steps} steps (bounded sample of the {args.pairs}-pair batch), sequential pairs "
              f"like the reference process, OpenMP({cores}) inside each stage")
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32/f64",
        "data": "synthetic", "config": workload_config(args, world),
        "cpu_baseline": {"value": val, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample},
        "cpu_best_case": {"value": best, "unit": UNIT, "cores": cores, "kind": "port",
                          "sample": f"{best_n} registrations, {cores} pairs in flight, one single-threaded oracle call per core"},
        "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "reference_sample_pairs_per_step": per_step,
        "note": "CPU restatement of the reference path (oracle/); the reference binary itself needs PCL/FLANN/pmc",
    }))


def workload_config(args, world):
    what = {"street": f"batch of {args.pairs} synthetic 64-ring pairs per GPU (BASELINE configs[2]; {world}x{args.pairs} global, 8 GPUs = configs[3])",
            "dense": f"batch of {args.pairs} synthetic 64-ring pairs per GPU, dense preset (L ~ 3 k correspondences per pair: the back end at "
                     f"BASELINE's stated size; {world}x{args.pairs} global)",
            "indoor": f"{args.pairs} dense indoor pairs per GPU per step (BASELINE configs[4]: ~500 k points per scan, 0.05 m voxel, ~50 k voxel "
                      f"points per cloud; {world}x{args.pairs} global)"}[args.scene]
    scan = "500 k uniformly distributed rays in a furnished 6 x 6 x 3 m room, 5 mm range noise" if args.scene == "indoor" else \
        "64 rings x 1800 azimuths, ~111k returns, ground flagged"
    return {"workload": what, "scene": args.scene,
            "pairs_per_gpu": args.pairs, "global_pairs": args.pairs * world, "scan": scan,
            "params": SCENES[args.scene]["what"],
            "l2": "inputs larger than L2 (~0.9 GB of raw scans per GPU per step vs 50 MB)" if args.scene != "indoor" else
                  f"inputs of {args.pairs} x 16 MB per step; L2 (50 MB) is flushed by the first pair's 0.8 GB of K6 operand traffic",
            "parallelism": f"dp{world}: independent pairs sharded across ranks, one NCCL all_gather of result records per step"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--scene", default="street", choices=sorted(SCENES))
    ap.add_argument("--pairs", type=int, default=256, help="pairs per GPU per step")
    ap.add_argument("--graph-L", type=int, default=3000, help="correspondences per set of the K8 roofline pass (0 = skip)")
    ap.add_argument("--slots", type=int, default=64, help="pairs per device wave (the lanes rotate over waves of this size)")
    ap.add_argument("--cpu-baseline-seconds", type=float, default=12.0)
    ap.add_argument("--ref-pairs-per-step", type=int, default=8)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--sync-steps", action="store_true", help="time the blocking qb200_register_batch per step (no batch k+1 under the tail of batch k)")
    ap.add_argument("--no-dense", action="store_true", help="skip the dense sub-measurement of the default (street) run")
    ap.add_argument("--cross-rank-pairs", type=int, default=8, help="pairs of the next rank every rank re-registers and compares (N > 1)")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's result records to DIR/<field>.npy (float64)")
    args = ap.parse_args()

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))

    if args.impl == "reference":
        run_reference(args, rank, world)
        return

    import torch
    import torch.distributed as dist
    from quatro_b200 import synth
    from quatro_b200.capi import Handle, Pair, RESULT_DTYPE, MEM_HOST, MEM_DEVICE

    torch.cuda.set_device(local_rank)
    if world > 1:
        # stdout carries exactly one JSON line: whatever NCCL logs (its version banner under NCCL_DEBUG=VERSION) goes to stderr
        os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    dev = torch.device("cuda", local_rank)
    P = args.pairs
    stream = torch.cuda.current_stream(dev)

    # ---- synthetic inputs: pinned host copy (e2e) and device-resident copy (value) ----
    def build_inputs(seeds):
        prs = gen_pairs(seeds, args.scene)
        total = sum(len(s) + len(t) for s, t in prs)
        host = torch.empty((total, 4), dtype=torch.float32).pin_memory()
        hv = host.numpy()
        offs, o = [], 0
        for s, t in prs:
            hv[o:o + len(s)] = s; offs.append((o, len(s))); o += len(s)
            hv[o:o + len(t)] = t; offs.append((o, len(t))); o += len(t)
        dvc = host.to(dev, non_blocking=False)
        n = len(prs)
        pa_h, pa_d = (Pair * n)(), (Pair * n)()
        for i in range(n):
            (so, sn), (to, tn) = offs[2 * i], offs[2 * i + 1]
            pa_h[i].src, pa_h[i].n_src, pa_h[i].tgt, pa_h[i].n_tgt = host.data_ptr() + so * 16, sn, host.data_ptr() + to * 16, tn
            pa_d[i].src, pa_d[i].n_src, pa_d[i].tgt, pa_d[i].n_tgt = dvc.data_ptr() + so * 16, sn, dvc.data_ptr() + to * 16, tn
        return prs, host, dvc, pa_h, pa_d, total

    def make_handle(scene):
        slots = min(args.slots, P, 2) if scene == "indoor" else min(args.slots, P)   # indoor: 64 MB of operand images per cloud
        hd = Handle(device=local_rank, max_batch_slots=slots, **SCENES[scene]["cfg"])
        hd.set_stream(stream.cuda_stream)
        return hd

    handle = make_handle(args.scene)
    # bind this rank's host thread to the GPU's NUMA node BEFORE the pinned input buffers are allocated and filled (first touch puts
    # the pages on the local socket): launches and host->device copies then never cross the inter-socket link
    numa_cores = handle.bind_numa()
    pairs, host, dvc, pa_host, pa_dev, total_pts = build_inputs(range(rank * P, rank * P + P))
    h2d_bytes = total_pts * 16
    d2h_bytes = P * RESULT_DTYPE.itemsize
    p = scene_params(args.scene)
    out = np.zeros(P, RESULT_DTYPE)
    out_all = np.zeros(world * P, RESULT_DTYPE) if world > 1 else None
    host_ms = {"enqueue": 0.0, "collective_wait": 0.0}
    if world > 1:
        # the path's only collective lives in the C++ library: one ncclAllGather of the result records per batch on the handle's
        # communication stream, deferred so that it overlaps the next step (qb200_register_batch_rank / qb200_comm_wait)
        uid = [Handle.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        handle.comm_init_rank(world, rank, uid[0])

    # Throughput mode (BASELINE configs[2]): the timed steps are a stream of batches.  On one GPU batch k+1 is queued
    # (qb200_register_batch_enqueue) before batch k has been collected, so the latency-bound tail of a batch runs under the copies
    # and front-end kernels of the next; qb200_register_batch_flush closes the timed region.  N > 1: the same through
    # qb200_register_batch_rank(defer = 2), which also starts batch k's all-gather while batch k+1 computes; qb200_comm_wait closes.
    # --sync-steps times the blocking call per step instead (N > 1: blocking local batch, deferred gather).
    mode = {"pipelined": not args.sync_steps}

    def step(hd, prm, pa, kind):
        t0 = time.perf_counter()
        if world > 1 and hd is handle:
            hd.register_batch_rank_raw(pa, P, prm, kind, out_all, defer=2 if mode["pipelined"] else 1)   # collects the PREVIOUS step's gather first
        elif mode["pipelined"]:
            hd.register_batch_enqueue_raw(pa, P, prm, kind, out)
        else:
            hd.register_batch_raw(pa, P, prm, kind, out)
        host_ms["enqueue"] += 1e3 * (time.perf_counter() - t0)

    def finish_gather():
        if world > 1:
            t0 = time.perf_counter()
            handle.comm_wait()
            host_ms["collective_wait"] += 1e3 * (time.perf_counter() - t0)
            out[:] = out_all[rank::world]

    def timed(hd, prm, pa, kind, steps, sampler=None):
        hd.register_batch_flush()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)
        if sampler:
            sampler.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = hd.launch_count()
        kms, kcalls, sms = np.zeros(2), np.zeros(2), np.zeros(8)
        e0.record(stream)
        for _ in range(steps):
            step(hd, prm, pa, kind)
            if not mode["pipelined"]:
                m, c = hd.kernel_ms()
                kms += m; kcalls += c; sms += hd.stage_ms()
        if mode["pipelined"]:
            t0 = time.perf_counter()
            hd.register_batch_flush()   # every record of every step is in place
            host_ms["enqueue"] += 1e3 * (time.perf_counter() - t0)
        if hd is handle:
            finish_gather()   # the last step's gather; qb200_comm_wait orders the handle's stream after it
        if mode["pipelined"]:
            m, c = hd.kernel_ms()
            kms += m; kcalls += c; sms += hd.stage_ms()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
        clocks = sampler.stop() if sampler else None
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()), hd.launch_count() - l0, kms, kcalls, sms, clocks

    def single_pair_latency(hd, prm):
        lat = []
        for i in range(12):
            a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a0.record(stream)
            hd.register_batch_raw(pa_host, 1, prm, MEM_HOST, out)
            a1.record(stream)
            torch.cuda.synchronize(dev)
            if i >= 2:
                lat.append(a0.elapsed_time(a1))
        return float(np.median(lat))

    def oracle_check(prm, res, seconds, max_pairs=64):
        """time the CPU oracle on the first pairs of this rank's batch and require identical records"""
        from oracle import Oracle
        o = Oracle()
        cores = o.set_num_threads(_host_threads())
        o.register_pair(pairs[0][0], pairs[0][1], prm)  # warm-up
        t0 = time.perf_counter(); n = 0
        while n < min(P, max_pairs) and time.perf_counter() - t0 < seconds:
            r, _ = o.register_pair(pairs[n][0], pairs[n][1], prm)
            g = res[n]
            assert (r.n_corr, r.clique_size, r.n_edges, r.max_core) == (g["n_corr"], g["clique_size"], g["n_edges"], g["max_core"]), \
                f"pair {n}: GPU result differs from the CPU oracle: {(r.n_corr, r.clique_size, r.n_edges, r.max_core)} vs {g}"
            assert np.allclose(np.asarray(g["T"]), np.array(r.T[:]), atol=1e-9), f"pair {n}: pose differs from the CPU oracle"
            n += 1
        return n / (time.perf_counter() - t0), n, cores

    for _ in range(args.warmup):
        step(handle, p, pa_dev, MEM_DEVICE)
    finish_gather()
    host_ms = {"enqueue": 0.0, "collective_wait": 0.0}
    dev_ms, launches, kms, kcalls, sms, clocks = timed(handle, p, pa_dev, MEM_DEVICE, args.steps, ClockSampler(local_rank) if rank == 0 else None)
    res_dev = out.copy()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, res_dev)
    out_all_dev = out_all.copy() if world > 1 else None
    host_dev = dict(host_ms)
    if world > 1:
        # every rank holds every record: the gathered copy of this rank's slice must be the local result
        assert out_all.reshape(P, world)[:, rank].tobytes() == out.tobytes()
    for _ in range(max(1, args.warmup // 2)):
        step(handle, p, pa_host, MEM_HOST)
    finish_gather()
    e2e_ms, _, _, _, _, _ = timed(handle, p, pa_host, MEM_HOST, args.steps)
    assert out.tobytes() == res_dev.tobytes(), "host-buffer and device-buffer runs disagree"

    value = world * P * args.steps / (dev_ms * 1e-3)
    e2e_value = world * P * args.steps / (e2e_ms * 1e-3)
    # the blocking call per step next to the pipelined stream of batches (same steps, same buffers)
    sync_steps = None
    if mode["pipelined"]:
        mode["pipelined"] = False
        sd_ms = timed(handle, p, pa_dev, MEM_DEVICE, args.steps)[0]
        se_ms = timed(handle, p, pa_host, MEM_HOST, args.steps)[0]
        mode["pipelined"] = True
        sync_steps = {"value": world * P * args.steps / (sd_ms * 1e-3), "e2e": world * P * args.steps / (se_ms * 1e-3), "unit": UNIT,
                      "what": "qb200_register_batch (blocking) per step instead of qb200_register_batch_enqueue per step + one flush"}

    # ---- N > 1: every rank re-registers the first k pairs of the NEXT rank and compares the bytes of the records ----
    cross = None
    if world > 1:
        k = max(1, min(args.cross_rank_pairs, P))
        nxt = (rank + 1) % world
        _, h2, d2, _, pa2, _ = build_inputs(range(nxt * P, nxt * P + k))
        mine = np.zeros(k, RESULT_DTYPE)
        handle.register_batch_raw(pa2, k, p, MEM_DEVICE, mine)
        # rank nxt's own records came with the library's gather: out_all[i * world + r]
        theirs = out_all_dev.reshape(P, world)[:k, nxt]
        same = bool(theirs.tobytes() == mine.tobytes())
        flag = torch.tensor([1 if same else 0], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        cross = {"pairs_per_rank": k, "identical_on_all_ranks": bool(flag.item() == 1),
                 "what": "rank r re-registered the first k pairs of rank (r+1) mod N and compared the result records byte for byte"}
        assert cross["identical_on_all_ranks"], "results depend on the rank that computed them"

    # BASELINE configs[1] (one pair on one GPU): latency of a single registration through the same call, host buffers
    single_ms = single_pair_latency(handle, p) if rank == 0 else None

    # ---- the dense workload (L ~ 3 k) as a sub-measurement of the default run: 1 GPU only, device-resident inputs ----
    dense = None
    if args.scene == "street" and world == 1 and not args.no_dense:
        pd = scene_params("dense")
        hd = make_handle("dense")
        for _ in range(2):
            step(hd, pd, pa_dev, MEM_DEVICE)
        d_ms, _, _, _, d_sms, _ = timed(hd, pd, pa_dev, MEM_DEVICE, 3)
        d_res = out.copy()
        d_single = single_pair_latency(hd, pd)
        hd.close()
        # one wave on one lane: the per-stage device times without overlap from other waves
        os.environ["QB200_LANES"] = "1"
        h1 = make_handle("dense")
        del os.environ["QB200_LANES"]
        n1 = min(args.slots, P)
        o1 = np.zeros(n1, RESULT_DTYPE)
        for _ in range(2):
            h1.register_batch_raw(pa_dev, n1, pd, MEM_DEVICE, o1)
        serial = h1.stage_ms().copy()
        h1.close()
        d_cpu = None
        if not args.no_cpu_baseline:
            v, n, cores = oracle_check(pd, d_res, min(args.cpu_baseline_seconds, 10.0), 32)
            d_cpu = {"value": v, "unit": UNIT, "cores": cores, "kind": "port",
                     "sample": f"first {n} pairs, sequential, OpenMP({cores}) inside stages; all {n} matched the GPU records (counters exact, pose <= 1e-9)"}
        names = ["h2d", "voxel", "fpfh", "match", "graph", "clique", "pose", "d2h"]
        dL = d_res["n_corr"].astype(np.float64)
        dense = {"config": {"workload": f"batch of {P} synthetic 64-ring pairs, dense preset", "params": SCENES["dense"]["what"]},
                 "value": P * 3 / (d_ms * 1e-3), "unit": UNIT, "ms_per_step": d_ms / 3, "steps": 3, "warmup": 2,
                 "mean_L": float(dL.mean()), "max_L": int(dL.max()), "mean_n_vox": float((d_res["n_src_vox"].mean() + d_res["n_tgt_vox"].mean()) / 2),
                 "mean_edges": float(d_res["n_edges"].mean()), "mean_clique": float(d_res["clique_size"].mean()),
                 "valid_pairs": int(d_res["valid"].sum()), "status_counts": {int(k): int(v) for k, v in zip(*np.unique(d_res["status"], return_counts=True))},
                 "stages_ms_per_step": {k: float(v / 3) for k, v in zip(names, d_sms)},
                 "stages_ms_one_wave_one_lane": {"pairs": n1, **{k: float(v) for k, v in zip(names, serial)}},
                 "single_pair_latency_ms": d_single, "cpu_baseline": d_cpu}

    # ---- pre-processing before the path (SURVEY 8f-1): ground removal + range-image sub-cluster rejection, per scan, host buffers ----
    preprocess = None
    if args.scene == "street" and world == 1 and rank == 0 and not args.no_dense:
        from quatro_b200.capi import default_patchwork_params, default_segment_params
        pp_, sp_ = default_patchwork_params(), default_segment_params()
        scans = [pairs[i][0] for i in range(min(8, P))]
        hp = Handle(device=local_rank, max_batch_slots=2)
        for sc in scans[:2]:
            hp.segment_cloud(hp.patchwork(sc, pp_)[1], sp_)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs = []
        for sc in scans:
            g_, ng_, _ = hp.patchwork(sc, pp_)
            outs.append((g_, ng_) + hp.segment_cloud(ng_, sp_))
        gpu_ms = (time.perf_counter() - t0) * 1e3 / len(scans)
        hp.close()
        cpu_ms, same = None, None
        if not args.no_cpu_baseline:
            from oracle import Oracle
            o_ = Oracle()
            t0 = time.perf_counter()
            same = True
            for sc, (g_, ng_, v_, ol_) in zip(scans, outs):
                og, ong, _ = o_.patchwork(sc, pp_)
                ov, ool = o_.segment_cloud(ong, sp_)
                same = same and np.array_equal(og, g_) and np.array_equal(ong, ng_) and np.array_equal(ov, v_) and np.array_equal(ool, ol_)
            cpu_ms = (time.perf_counter() - t0) * 1e3 / len(scans)
        preprocess = {"what": "qb200_patchwork + qb200_segment_cloud per scan through the C-ABI, host buffers in and out (the reference's STEP 2 / STEP 3, "
                              "examples/run_global_registration.cpp:136-162); wall clock per scan, blocking calls",
                      "scans": len(scans), "ms_per_scan": gpu_ms, "cpu_oracle_ms_per_scan": cpu_ms, "identical_to_oracle": same,
                      "mean_points": float(np.mean([len(x) for x in scans])), "mean_ground": float(np.mean([len(x[0]) for x in outs])),
                      "mean_valid_segment_points": float(np.mean([len(x[2]) for x in outs]))}

    if rank == 0:
        peaks = load_peaks()
        nA, nB, L = res_dev["n_src_vox"].astype(np.float64), res_dev["n_tgt_vox"].astype(np.float64), res_dev["n_corr"].astype(np.float64)
        # K6: 66 flop per (src,tgt) descriptor pair (the 2*33 of the ||a||^2+||b||^2-2ab contraction, SURVEY.md 8d)
        match_flops_step = float((66.0 * nA * nB).sum())
        match_ms_launch = kms[0] / max(kcalls[0], 1)
        launches_per_step = kcalls[0] / args.steps
        match_tflops = match_flops_step / launches_per_step / (match_ms_launch * 1e-3) / 1e12 if match_ms_launch > 0 else 0.0
        # K8: algorithmic bytes = 2*L*16 (matched points) + L*ceil(L/32)*4 (bit adjacency) + 4L (degrees)
        graph_bytes_step = float((2 * L * 16 + L * np.ceil(L / 32) * 4 + 4 * L).sum())
        graph_ms_launch = kms[1] / max(kcalls[1], 1)
        graph_gbs = graph_bytes_step / (kcalls[1] / args.steps) / (graph_ms_launch * 1e-3) / 1e9 if graph_ms_launch > 0 else 0.0
        step_ms = dev_ms / args.steps
        flops_launch = match_flops_step / max(launches_per_step, 1)
        tf32_peak = peaks["bf16_tflops"] / 2.0
        roofline = {"kernel": "tc_nn_kernel (K6: wgmma 3xTF32 filter of the N_src x N_tgt x 33 distance matrix + in-kernel exact fp32 evaluation)",
                    "bound": "tensor", "achieved": match_tflops, "peak": peaks["bf16_tflops"], "unit": "TFLOP/s",
                    "frac": match_tflops / peaks["bf16_tflops"],
                    "frac_of_tf32_peak": match_tflops / tf32_peak,
                    "tf32_peak": tf32_peak, "tf32_peak_source": "half of the bf16 peak (the kernel's MMAs are TF32; nominal dense tf32 = bf16 / 2)",
                    "traffic": None,
                    "algorithmic_bytes_per_launch": float(((nA + nB) * 132.0).sum()) / max(launches_per_step, 1),
                    "peak_source": peaks["source"] + ", burst bf16",
                    "launch_ms": match_ms_launch, "launches_per_step": launches_per_step, "share_of_step": float(kms[0] / args.steps / step_ms),
                    "flops_per_launch": flops_launch,
                    "note": "achieved = 66 flop per descriptor pair (algorithmic, all n_src x n_tgt pairs) / launch time measured with CUDA events inside the timed steps (other lanes' kernels share the SMs meanwhile); the kernel skips most tiles by a norm lower bound and runs 3xTF32 on K padded to 40 on the rest (DESIGN.md 5.1)"}
        roofline_graph = {"kernel": "tim_graph_kernel (K8)", "bound": "hbm", "achieved": graph_gbs, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                          "frac": graph_gbs / peaks["hbm_gbs"], "traffic": None, "launch_ms": graph_ms_launch,
                          "bytes_per_launch": graph_bytes_step / max(kcalls[1] / args.steps, 1), "mean_L": float(L.mean()),
                          "note": "fp32-pipe bound at algorithmic-minimum bytes (SURVEY.md 8d): ~18 instructions per pair test vs 0.27 B per pair"}
        # K8 at the size BASELINE's configs name (~3k correspondences per pair): 32 precomputed correspondence sets through
        # qb200_solve_batch (device-resident), tim_graph_kernel timed with CUDA events inside the call
        roofline_graph_3k = None
        if args.graph_L > 0:
            gsets, keep = [], []
            for i in range(32):
                a4, b4, _, _ = synth.matched_pairs(7000 + i, args.graph_L, inlier_ratio=0.03, noise=0.04)
                ta, tb = torch.from_numpy(np.ascontiguousarray(a4)).to(dev), torch.from_numpy(np.ascontiguousarray(b4)).to(dev)
                keep.append((ta, tb))
                gsets.append((ta.data_ptr(), tb.data_ptr(), len(a4)))
            torch.cuda.synchronize(dev)
            hg = Handle(device=local_rank, max_batch_slots=32)
            hg.set_stream(stream.cuda_stream)
            hg.solve_batch(gsets, p, kind=MEM_DEVICE)  # warm-up
            gms, gcalls, gst = 0.0, 0, np.zeros(8)
            for _ in range(5):
                rg = hg.solve_batch(gsets, p, kind=MEM_DEVICE)
                m, c = hg.kernel_ms()
                gms += float(m[1]); gcalls += int(c[1]); gst += hg.stage_ms()
            hg.close()
            Lg = float(args.graph_L)
            g_bytes = 32 * (2 * Lg * 16 + Lg * np.ceil(Lg / 32) * 4 + 4 * Lg)
            g_ms = gms / max(gcalls, 1)
            g_pairs = 32 * Lg * (Lg - 1) / 2
            # fp32 view: 14 fma-pipe operations (9 FFMA + 5 FADD) per pair test against SMs x 128 lanes x clock (1 op/lane/clk),
            # at the largest SM clock sampled during the timed steps (H100 SXM boost clock when nvidia-smi is unavailable)
            n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
            sm_hz = ((clocks or {}).get("sm_max_mhz") or 1980.0) * 1e6
            fp32_ops_peak = n_sm * 128 * sm_hz
            roofline_graph_3k = {"kernel": "tim_graph_kernel (K8)", "bound": "fp32 pipe (named bound); hbm fraction reported as BASELINE asks",
                                 "achieved": g_bytes / (g_ms * 1e-3) / 1e9, "peak": peaks["hbm_gbs"],
                                 "unit": "GB/s", "frac": g_bytes / (g_ms * 1e-3) / 1e9 / peaks["hbm_gbs"],
                                 "traffic": None,
                                 "launch_ms": g_ms,
                                 "L": int(Lg), "sets_per_launch": 32, "bytes_per_launch": g_bytes, "pair_tests_per_s": g_pairs / (g_ms * 1e-3),
                                 "fp32_frac": 14.0 * g_pairs / (g_ms * 1e-3) / fp32_ops_peak,
                                 "fp32_frac_note": f"14 fma-pipe operations per pair test (9 FFMA + 5 FADD) x pair tests/s / ({n_sm} SMs x 128 lanes x {sm_hz / 1e9:.3f} GHz)",
                                 "solve_batch_stage_ms": {"graph": float(gst[4] / 5), "clique": float(gst[5] / 5), "pose": float(gst[6] / 5)},
                                 "valid_sets": int(rg["valid"].sum()),
                                 "note": "algorithmic-minimum bytes (0.27 B per pair test) against ~18 fp32 instructions per pair test: the kernel is bound by the fp32 pipe, pair_tests_per_s is the meaningful rate"}
        cpu = best = None
        if not args.no_cpu_baseline:
            v, n, cores = oracle_check(p, res_dev, args.cpu_baseline_seconds)
            cpu = {"value": v, "unit": UNIT, "cores": cores, "kind": "port",
                   "sample": f"first {n} pairs of rank 0's batch, sequential pairs, OpenMP({cores}) inside stages; all {n} matched the GPU records"}
            bv, bn = cpu_pair_parallel(pairs[:64], p, cores, min(8.0, args.cpu_baseline_seconds))
            best = {"value": bv, "unit": UNIT, "cores": cores, "kind": "port",
                    "sample": f"{bn} registrations, {cores} pairs in flight, one single-threaded oracle call per core (best-case CPU, SURVEY.md 8d)"}
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": step_ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32 (front end, match, graph filter) / f64 (graph boundary, GNC, COTE)",
            "data": "synthetic", "config": workload_config(args, world),
            "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": d2h_bytes, "ms_per_step": e2e_ms / args.steps},
            "gpu_launches": int(launches), "clocks": clocks, "roofline": roofline, "roofline_graph": roofline_graph,
            "roofline_graph_3k": roofline_graph_3k, "cpu_baseline": cpu, "cpu_best_case": best, "dense": dense, "preprocess": preprocess, "cross_rank_check": cross,
            "stages_ms_per_step": {k: float(v / args.steps) for k, v in zip(["h2d", "voxel", "fpfh", "match", "graph", "clique", "pose", "d2h"], sms)},
            "valid_pairs": int(res_dev["valid"].sum()), "mean_n_vox": float((nA.mean() + nB.mean()) / 2), "mean_L": float(L.mean()),
            "mean_clique": float(res_dev["clique_size"].mean()),
            "single_pair_latency_ms": single_ms,
            "steps_mode": ("pipelined: every step is one qb200_register_batch_enqueue of the whole batch, one qb200_register_batch_flush before the "
                           "closing event (throughput mode: the tail of batch k overlaps the copies and front end of batch k+1)"
                           if mode["pipelined"] else "blocking call per step"),
            "sync_steps": sync_steps,
            "host_ms_per_step_rank0": {"enqueue": host_dev["enqueue"] / args.steps, "collective_wait": host_dev["collective_wait"] / args.steps,
                                       "device": step_ms, "numa_cores_bound": numa_cores,
                                       "what": "host time inside qb200_register_batch(_rank) per step; time blocked in qb200_comm_wait (the deferred "
                                               "gather of the last step only); device time per step (CUDA events, max over ranks)"},
        }
        print(json.dumps(line))
    handle.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
