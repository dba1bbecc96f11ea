#!/usr/bin/env python
"""bench.py — scans/sec of the LiLi-OM per-scan hot path on H100 (BASELINE.json metric).

One "step" = one scan through the hot path:
    feature extraction (raw sweep) -> VoxelGrid(0.4) of the surf features -> ITERS x
    [5-NN in the voxel map + plane fit + residual/Jacobian + 27-scalar reduce + 6x6 solve + pose update]
    (+ per-scan map maintenance in the streamed workload: push a frame, re-filter and re-index the local map)

N = 1 : BASELINE.json configs[1] — 24k-pt Livox-Horizon sweep, 1 M-pt voxel map, 10 GN iterations, map pre-built
        (--workload rot: configs[2], 130k-pt HDL-64E sweep through the LiLi-OM-ROT extractor, 2 M-pt map).
N > 1 : BASELINE.json configs[4] (--multi sharded, default) — ONE scan stream: 130k-pt HDL-64E sweep, 10 M-pt local map kept as a
        FIFO of 20 frames and SHARDED by voxel-block hash across the GPUs (halo replicated), 10 GN iterations with one exchange
        of the 29 normal-equation scalars per iteration (fused into the GN kernel over NVLink peer memory; NCCL all-reduce
        with LILIOM_BENCH_NCCL=1), and the reference's per-scan map maintenance INSIDE the step (L/src/LidarOdometry.cpp:
        280-323, 490: push the frame, concatenate, VoxelGrid(0.4), rebuild the search structure) — the part that shards.
        Strong scaling: the line also carries the same workload on one GPU, measured in the same run (`same_workload_1gpu`).
        --multi replicas: every GPU runs the N = 1 workload on its own scan stream (no collective, weak scaling); the
        sharded line reports it as a secondary key (`replicas`).

value  : scans/s with the sweep already resident in HBM (only the 56-byte pose returns to the host).
e2e    : scans/s through the reference-facing calls with HOST (pinned) buffers — Preprocessing node call (H2D raw sweep,
         D2H the three published clouds) + LidarOdometry node call (H2D surf cloud, D2H pose + surf_last_ds)
         (+ H2D of the pushed frame in the streamed workload).
roofline: kNN+Jacobian kernel — algorithmic bytes per SURVEY.md §8(d), B_q = 16 + 27*8 + 16*C-bar per query and pass with
         C-bar = points in the query's 27 cells (counted by liliom_knn_block_stats), over the CUDA-event duration of a pass,
         against the measured HBM peak.  The search prunes; `examined` carries the same figure on the bytes actually fetched.
cpu_baseline: the CPU oracle (restatement of the reference, oracle/) on the host cores, bounded sample, 1 thread.
--impl reference: the same workload on the CPU oracle with the host threads (the reference itself cannot be built here:
         needs ROS/PCL/Eigen/Ceres).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

ITERS = 10
N_FRAMES = 20
KTIME_EVERY = 5
SHARD_BLOCK_M = 64
METRIC = "scans/sec (24k-pt sweep vs 1M-pt map); kNN+Jacobian HBM GB/s vs peak"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--multi", default="sharded", choices=["sharded", "replicas"])
    ap.add_argument("--map-points", type=int, default=0, help="override the map size")
    ap.add_argument("--sweeps", type=int, default=8, help="distinct synthetic sweeps cycled through the steps")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--e2e", default="two-nodes", choices=["two-nodes", "sequential"],
                    help="e2e leg at N = 1: two concurrent node threads (reference architecture, default) or one thread calling both nodes in turn")
    ap.add_argument("--dense-queries", action="store_true", help="roofline micro-run: every surf feature is a query (no scan DS)")
    ap.add_argument("--no-dense-probe", action="store_true", help="skip the dense-query probes that annotate roofline.dense_probe")
    ap.add_argument("--no-extra-legs", action="store_true", help="N > 1: skip the same-workload-on-one-GPU and replicas legs")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="after the timed steps, write what the last timed step of each leg returned (poses, query count, the clouds "
                         "of the end-to-end leg) as DIR/<name>.npy, float32 / float64, rank 0 only")
    ap.add_argument("--workload", default="", choices=["", "horizon", "rot", "stream"],
                    help="horizon: configs[1] (default at N = 1); rot: configs[2]; stream: configs[4]'s streamed workload "
                         "(130k sweep, 10 M-pt map as 20 frames, map maintenance in the step; default at N > 1, also runs at N = 1)")
    return ap.parse_args()


def measured_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3; not measured)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed regions (the profiling recipe's clocks line): ONE `nvidia-smi
    --query-gpu=... -lms` process, started well before the first timed step and stopped after the last, its rows stamped on
    arrival; summary() keeps the rows that fall inside the window.  (One looping process rather than one process per sample:
    every nvidia-smi start-up initialises NVML and takes driver locks for several ms, which a 20-step timed region of ~10 ms
    would feel as launch latency.)  Rank 0 only: one poller per node is enough."""
    PERIOD_MS = 25

    def __init__(self, index: int, enabled: bool = True):
        self.index = index
        self.enabled = enabled
        self.rows = []            # (monotonic arrival time, fields)
        self.t0 = self.t1 = None
        self._p = None
        self._t = None

    def start(self):
        if not self.enabled or self._p is not None:
            return self
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        try:
            self._p = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}", "--format=csv,noheader,nounits",
                                        "-lms", str(self.PERIOD_MS)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, bufsize=1)
        except Exception:
            self._p = None
            return self

        def reader():
            try:
                for ln in self._p.stdout:
                    ln = ln.strip()
                    if ln:
                        self.rows.append((time.monotonic(), [x.strip() for x in ln.split(",")]))
            except Exception:
                pass
        self._t = threading.Thread(target=reader, daemon=True)
        self._t.start()
        return self

    def __enter__(self):                      # the window: the timed regions
        self.start()
        self.t0 = time.monotonic()
        return self

    def __exit__(self, *a):
        self.t1 = time.monotonic()

    def stop(self):
        if self._p is not None:
            time.sleep(2.5 * self.PERIOD_MS * 1e-3)           # let the sample after the window arrive
            try:
                self._p.terminate()
                self._p.wait(timeout=3)
            except Exception:
                try:
                    self._p.kill()
                except Exception:
                    pass
            if self._t:
                self._t.join(timeout=3)
            self._p = None

    def summary(self):
        self.stop()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        t0 = self.t0 if self.t0 is not None else float("-inf")
        t1 = self.t1 if self.t1 is not None else float("inf")
        slack = 1.5 * self.PERIOD_MS * 1e-3                    # a row is stamped when it ARRIVES, up to one period after its sample
        inside = [r for t, r in self.rows if t0 <= t <= t1 + slack]
        for r in inside:
            try:
                sm.append(float(r[0])); mx.append(float(r[1]))
                for k, nm in enumerate(names):
                    if r[2 + k].lower().startswith("active"):
                        reasons.add(nm)
            except Exception:
                pass
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": float(max(mx)) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm), "period_ms": self.PERIOD_MS}


def resolve_e2e(run_two_nodes, over_ranks, ms_seq, last_seq):
    """The optional two-node e2e leg, fail-safe: if it raises on ANY rank, every rank reports the one-thread figure instead (the
    decision is taken on the gathered per-rank times, so all ranks take the same branch and the collectives stay matched).
    Returns (ms over ranks, last result, error text or None)."""
    err = None
    try:
        ms_local, last = run_two_nodes()
    except Exception as ex:      # noqa: BLE001 — an optional leg must not cost the whole bench line
        ms_local, last, err = float("nan"), None, f"{type(ex).__name__}: {str(ex)[:200]}"
    _, per = over_ranks(ms_local)
    if any(p != p for p in per):
        return ms_seq, last_seq, (err or "the two-node leg failed on another rank")
    return max(per), last, None


def run_two_stage_pipeline(total, warmup, nbuf, stage_a, stage_b, on_start, on_end, timeout_s=120.0):
    """Two host threads joined by a bounded queue (nbuf buffers in flight).  stage_a(k, buf) -> item,
    stage_b(k, buf, item).  on_start() runs on thread A after both stages have fully drained the `warmup`
    steps; on_end() runs on thread B after the last step.  Any exception / timeout is re-raised in the caller."""
    import queue
    free_q, work_q = queue.Queue(), queue.Queue()
    for b in range(nbuf):
        free_q.put(b)
    gate = threading.Barrier(2, timeout=timeout_s)
    errors = []

    def a_thread():
        try:
            for k in range(total):
                if k == warmup:
                    gate.wait()          # thread B arrives here after finishing step warmup-1
                    on_start()
                b = free_q.get(timeout=timeout_s)
                work_q.put((k, b, stage_a(k, b)))
        except BaseException as e:       # noqa: BLE001
            errors.append(e)
            gate.abort()
        finally:
            work_q.put(None)

    def b_thread():
        try:
            if warmup == 0:
                gate.wait()
            while True:
                item = work_q.get(timeout=timeout_s)
                if item is None:
                    break
                k, b, payload = item
                stage_b(k, b, payload)
                free_q.put(b)
                if k == warmup - 1:
                    gate.wait()
            on_end()
        except BaseException as e:       # noqa: BLE001
            errors.append(e)
            gate.abort()
            free_q.put(0)

    ta = threading.Thread(target=a_thread, daemon=True); tb = threading.Thread(target=b_thread, daemon=True)
    ta.start(); tb.start()
    ta.join(timeout_s * 4); tb.join(timeout_s * 4)
    if errors:
        raise errors[0]
    if ta.is_alive() or tb.is_alive():
        raise RuntimeError("two-stage pipeline did not finish")


# ---------------------------------------------------------------------------------------------- workloads
def resolve_workload(args, world):
    """(kind, n_map): horizon = configs[1], rot = configs[2], stream = configs[4]'s streamed workload."""
    sharded = world > 1 and args.multi == "sharded"
    kind = args.workload or ("stream" if sharded else "horizon")
    n_map = args.map_points or {"horizon": 1_000_000, "rot": 2_000_000, "stream": 10_000_000}[kind]
    return kind, n_map


def make_workload(kind: str, n_map: int, n_sweeps: int):
    from liliom_b200 import synth
    m, _ = synth.make_map(n_map)
    T0 = synth.default_true_pose()
    sweeps = []
    for k in range(n_sweeps):
        T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k       # sensor advancing through the block
        if kind == "horizon":
            pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        else:
            pts, q = synth.make_hdl64_sweep(T, seed=2 + k)
        sweeps.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))
    return m, sweeps


def make_frames(m, PT):
    """The streamed workload's local map as the reference holds it: a FIFO of N_FRAMES world-frame clouds (here: equal
    slabs of the synthetic map along x, oldest first) whose concatenation, VoxelGrid-filtered, is the map."""
    order = np.argsort(m[:, 0], kind="stable")
    frames = []
    per = (len(m) + N_FRAMES - 1) // N_FRAMES
    for k in range(N_FRAMES):
        idx = order[k * per:(k + 1) * per]
        f = np.zeros(len(idx), PT)
        f["x"] = m[idx, 0]; f["y"] = m[idx, 1]; f["z"] = m[idx, 2]; f["w"] = 1.0
        frames.append(f)
    return frames


def workload_name(kind, n_returns, n_map):
    if kind == "rot":
        return f"130k-pt HDL-64E sweep ({n_returns} returns, LiLi-OM-ROT extractor, ds_rate 4) vs {n_map}-pt voxel map, {ITERS} GN iters"
    if kind == "stream":
        return (f"streamed: 130k-pt HDL-64E sweep ({n_returns} returns, LiLi-OM-ROT extractor, ds_rate 4) vs {n_map}-pt local map held as "
                f"{N_FRAMES} frames, {ITERS} GN iters, then per-scan map maintenance (push frame, concatenate, VoxelGrid 0.4, re-index) inside the step")
    return f"24k-pt Livox-Horizon sweep ({n_returns} returns) vs {n_map}-pt voxel map, {ITERS} GN iters"


def config_dict(kind, n_returns, n_map, world, multi):
    """The `config` object — the SAME keys and values in both arms (ours / reference)."""
    return {"workload": workload_name(kind, n_returns, n_map), "kind": kind, "map_points": n_map, "iters": ITERS,
            "map_frames": N_FRAMES if kind == "stream" else 0,
            "multi": ("single" if world == 1 else multi), "n_gpus": world,
            "l2": "GPU arm: a 256 MB buffer is written between timed steps (L2 flushed), each step timed with its own CUDA-event pair on the "
                  "launch stream; CPU arm: wall clock around the timed steps"}


# ---------------------------------------------------------------------------------------------- CPU oracle legs
class CpuWorkload:
    """The oracle (oracle/, test infrastructure) running one scan of the workload — the cpu_baseline leg and --impl reference."""

    def __init__(self, kind, m, sweeps):
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import oracle_lib as O
        self.O, self.kind, self.sweeps = O, kind, sweeps
        t0 = time.perf_counter()
        if kind == "stream":
            self.frames = make_frames(m, O.PT32)
            self.map4 = self._filter_and_index()          # as the reference: VoxelGrid of the concatenation, kd-tree over it
        else:
            self.map4 = m
            self.tree = O.KdTree(m)
        self.t_setup = time.perf_counter() - t0

    def _filter_and_index(self):
        O = self.O
        ds = O.voxelgrid(np.concatenate(self.frames), 0.4)                 # L/src/LidarOdometry.cpp:301-302, 316-317
        m4 = np.ones((len(ds), 4), np.float32)
        m4[:, 0] = ds["x"]; m4[:, 1] = ds["y"]; m4[:, 2] = ds["z"]
        self.tree = O.KdTree(m4)                                           # :490
        return m4

    def scan(self, k, nthreads):
        O, sw = self.O, self.sweeps[k % len(self.sweeps)]
        if sw["pts"].dtype.itemsize == 32:      # ROT package
            rc, surf, edge, cut, _, _ = O.extract_rot(sw["pts"], sw["q"], (1.0, 0, 0, 0), 64, 4)
        else:
            surf, edge, cut = O.extract_horizon(sw["pts"], sw["q"])
        ds = O.voxelgrid(surf, 0.4)
        rc, pose, st = O.scan_to_map_gn(self.tree, ds, sw["guess"], ITERS, nthreads)
        if self.kind == "stream":               # per-scan map maintenance: pop the oldest frame, push one, re-filter, re-index
            ident = np.array([1.0, 0, 0, 0, 0, 0, 0])
            f = self.frames.pop(0)
            self.frames.append(O.transform_cloud(f, ident))                # :246-278 on the pushed frame
            self.map4 = self._filter_and_index()
        return pose, len(ds)


def run_reference(args):
    """--impl reference: the oracle port on the host cores (rank 0 only)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    world = int(os.environ.get("WORLD_SIZE", "1"))
    kind, n_map = resolve_workload(args, world)
    m, sweeps = make_workload(kind, n_map, min(args.sweeps, 4))
    W = CpuWorkload(kind, m, sweeps)
    cores = os.cpu_count() or 1
    os.environ.setdefault("OMP_WAIT_POLICY", "passive")
    # thread count: median of PROBE scans per candidate (OpenMP over the queries can lose on shared hosts); 1 thread is the
    # reference's own architecture and is always reported beside the best
    heavy = kind == "stream"
    PROBE = 1 if heavy else 5
    cands = sorted({1, 4, 8, 16, 32, cores} & set(range(1, cores + 1))) if not heavy else sorted({1, min(16, cores)})
    probe = {}
    W.scan(0, 1)                                            # first-touch warm-up, not timed
    for nt in cands:
        ts = []
        for k in range(PROBE):
            t0 = time.perf_counter(); W.scan(k, nt); ts.append(time.perf_counter() - t0)
        probe[nt] = float(np.median(ts))
    best_nt = min(probe, key=probe.get)
    warm = max(args.warmup, 3) if not heavy else 1
    steps = max(1, min(args.steps, int(45.0 / max(probe[best_nt], 1e-3))))
    for k in range(warm):
        W.scan(k, best_nt)
    t0 = time.perf_counter()
    for k in range(steps):
        W.scan(k, best_nt)
    dt = time.perf_counter() - t0
    val = steps / dt
    sample = (f"{steps} scans (extract + VoxelGrid + {ITERS} GN iters" + (", + map maintenance: VoxelGrid of the 20-frame concatenation and kd-tree build per scan" if heavy else
              f", kd-tree prebuilt in {W.t_setup:.2f}s, excluded — the reference rebuilds it per scan, L/src/LidarOdometry.cpp:490") + ")")
    cfg = config_dict(kind, len(sweeps[0]["pts"]), n_map, world, args.multi)
    line = {"impl": "reference", "metric": METRIC, "value": val, "unit": "scans/s", "n_gpus": args.gpus, "steps": steps,
            "warmup": warm, "ms_per_step": 1e3 * dt / steps, "higher_is_better": True,
            "scaling": "strong" if (world > 1 and args.multi == "sharded") else "weak",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic", "config": cfg,
            "impl_note": "CPU oracle port of the reference path (oracle/): the reference itself needs ROS/PCL/Eigen/Ceres and cannot be built in "
                         "this image; OpenMP over the queries, thread count = best median of the probe scans; extraction and VoxelGrid are "
                         "single-threaded as in the reference",
            "threads_probe_s_per_scan": {str(k): v for k, v in probe.items()},
            "one_thread_value": 1.0 / probe[1],
            "cpu_baseline": {"value": val, "unit": "scans/s", "cores": best_nt, "kind": "port", "sample": sample},
            "e2e": {"value": val, "unit": "scans/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def cpu_baseline_leg(kind, m, sweeps):
    W = CpuWorkload(kind, m, sweeps)
    W.scan(0, 1)
    n = 0
    t0 = time.perf_counter()
    while True:
        W.scan(n, 1)
        n += 1
        if time.perf_counter() - t0 > 10.0:
            break
    dt = time.perf_counter() - t0
    return {"value": n / dt, "unit": "scans/s", "cores": 1, "kind": "port",
            "sample": f"{n} scans in {dt:.1f}s, 1 thread (the reference nodes are single-threaded)"
                      + (", map maintenance (VoxelGrid + kd-tree build) included" if kind == "stream" else
                         ", kd-tree build EXCLUDED (the reference rebuilds it per scan, L/src/LidarOdometry.cpp:490: with it the CPU figure is lower)")}


def dump_outputs(d, arrays):
    """--dump-outputs: one DIR/<name>.npy per array (a few MB in all: the clouds of one sweep), so that two builds can be compared
    output for output on the same seeded inputs."""
    os.makedirs(d, exist_ok=True)
    for name, a in arrays.items():
        assert a.dtype in (np.float32, np.float64), (name, a.dtype)
        np.save(os.path.join(d, name + ".npy"), a)


# ---------------------------------------------------------------------------------------------- GPU legs
def main():
    args = parse()
    if args.impl == "reference":
        run_reference(args)
        return
    import torch
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device (no CPU fallback); use --impl reference for the CPU oracle")
    torch.cuda.set_device(local_rank)
    if world > 1:
        # One launch-latency-bound process per GPU: keep each on the host cores next to its GPU (a doorbell rung across sockets
        # costs more than the kernels of a 0.2 ms scan save).  Best effort; the line reports what the process ended up with.
        try:
            import pynvml
            pynvml.nvmlInit()
            pynvml.nvmlDeviceSetCpuAffinity(pynvml.nvmlDeviceGetHandleByIndex(local_rank))
            os.environ["LILIOM_BENCH_AFFINITY"] = "nvml"
        except Exception as e:      # noqa: BLE001
            os.environ["LILIOM_BENCH_AFFINITY"] = "unchanged (" + type(e).__name__ + ")"
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    note = None
    while True:
        again = bench_body(args, note)
        if again is None:
            break
        args.multi, args.workload, note = "replicas", "", again      # the sharded path failed its pre-flight on some rank: report replicas, say why
    if world > 1:
        dist.destroy_process_group()


def bench_body(args, fallback_note=None):
    import torch
    import liliom_b200 as L
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    multi = world > 1
    if multi:
        import torch.distributed as dist
    sharded = multi and args.multi == "sharded"
    kind, n_map = resolve_workload(args, world)
    stream_wl = kind == "stream"
    rot = kind != "horizon"
    steps = args.steps
    warmup = max(args.warmup, 3)

    m, sweeps = make_workload(kind, n_map, args.sweeps)
    if multi and not sharded:     # replicas: every rank gets its own scan stream
        sweeps = sweeps[rank % len(sweeps):] + sweeps[:rank % len(sweeps)]

    prm = L.default_params(1 if rot else 0)
    PT = L.PT32 if rot else L.PT48
    psz = PT.itemsize
    if args.dense_queries:
        prm.leaf_scan = 0.0        # no scan down-sampling: every surf feature is a query (roofline micro-run)
    stream = torch.cuda.Stream()
    clk = ClockSampler(local_rank, enabled=(rank == 0)).start()      # running long before the first timed step
    ident = np.array([1.0, 0, 0, 0, 0, 0, 0])
    use_nccl_exchange = bool(os.environ.get("LILIOM_BENCH_NCCL"))

    def new_context(with_comm: bool):
        cx = L.Context(prm, device=local_rank)
        cx.set_stream(stream.cuda_stream)
        if with_comm:
            uid = [L.comm_get_unique_id() if rank == 0 else None]
            dist.broadcast_object_list(uid, src=0)
            cx.comm_init(uid[0], world, rank)
            if stream_wl:
                cx.comm_set_shard_block(SHARD_BLOCK_M)       # a 1.2 km map: 64 m cubes keep the replicated rim near 10 %
            if not use_nccl_exchange:     # fused exchange over NVLink peer memory: one launch per scan and rank, no collective call per iteration
                hs = [None] * world
                dist.all_gather_object(hs, cx.comm_peer_export())
                cx.comm_peer_attach(hs, rank)
        return cx

    # ---- the streamed workload's frames: device-resident (resident leg) and pinned host (e2e leg)
    frames_host, frames_dev = [], []
    if stream_wl:
        for f in make_frames(m, PT):
            th = torch.from_numpy(f.view(np.uint8).reshape(-1)).pin_memory()
            frames_host.append(th.numpy().view(PT))
            frames_dev.append(th.to("cuda", non_blocking=True))
        torch.cuda.synchronize()

    def install_map(cx):
        if stream_wl:
            cx.map_clear()
            for fd in frames_dev:
                cx.map_push_frame_device(fd.data_ptr(), fd.numel() // psz, ident)
            return cx.map_rebuild()
        cx.map_set_points(m)
        return len(m)

    def preflight(cx):
        """Two scans of the sharded step before anything is timed (first call: per-iteration launches, second: the single
        persistent launch): every rank must come back with a finite pose, and all ranks with the same one."""
        ok, why = 1, ""
        try:
            sw = sweeps[0]
            for _ in range(2):
                cx.upload_scan(sw["pts"])
                cx.extract_resident(sw["q"])
                pose, _, _ = cx.odometry_resident(sw["guess"], ITERS, mode=L.MODE_GN, want_stats=False)
            if not np.all(np.isfinite(pose)):
                ok, why = 0, "non-finite pose"
        except Exception as e:      # noqa: BLE001
            ok, why, pose = 0, str(e)[:160], np.zeros(7)
        t = torch.tensor([float(ok)] + [float(x) if np.isfinite(x) else 0.0 for x in pose], dtype=torch.float64, device="cuda")
        lo, hi = t.clone(), t.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        if float(lo[0].item()) < 1.0:
            return False, why or "another rank failed"
        if float((hi[1:] - lo[1:]).abs().max().item()) != 0.0:
            return False, "ranks disagree on the pose"
        return True, ""

    exchange_note = None
    if sharded:
        ctx, good = None, False
        for mode in (["nccl"] if use_nccl_exchange else ["peer", "nccl"]):
            use_nccl_exchange = mode == "nccl"
            try:
                ctx = new_context(True)
                n_map_installed = install_map(ctx)
                good, why = preflight(ctx)
            except Exception as e:      # noqa: BLE001
                good, why = False, str(e)[:160]
            if good:
                break
            exchange_note = f"{mode} exchange failed its pre-flight ({why})"
            if ctx is not None:
                try:
                    ctx.close()
                except Exception:      # noqa: BLE001
                    pass
                ctx = None
        if not good:
            return "sharded path failed its pre-flight on this box (" + (exchange_note or "") + "); replicas reported instead"
    else:
        ctx = new_context(False)
        n_map_installed = install_map(ctx)
    # an event pair around the kNN+Jacobian kernel on every KTIME_EVERY-th scan (stride co-prime with the number of distinct sweeps):
    # each pair costs the step ~8-10 us of dependent stream latency, so timing every scan would tax the number it explains
    ctx.set_kernel_timing(KTIME_EVERY)

    # pinned host buffers for the e2e leg (the contract: inputs come from pinned host memory)
    pin_sweeps = []
    for sw in sweeps:
        t = torch.from_numpy(sw["pts"].view(np.uint8).reshape(-1)).pin_memory()
        pin_sweeps.append(t.numpy().view(PT))
    cap = max(len(s["pts"]) for s in sweeps)
    out_surf = torch.empty(cap * psz, dtype=torch.uint8).pin_memory().numpy().view(PT)
    out_edge = torch.empty(cap * psz, dtype=torch.uint8).pin_memory().numpy().view(PT)
    out_cut = torch.empty(cap * psz, dtype=torch.uint8).pin_memory().numpy().view(PT)
    out_ds = torch.empty(cap * psz, dtype=torch.uint8).pin_memory().numpy().view(PT)

    def extract_host(cx, i, out):
        if rot:
            return cx.extract_rot(pin_sweeps[i], sweeps[i]["q"], out=out)
        return cx.extract_horizon(pin_sweeps[i], sweeps[i]["q"], out=out)
    pose_buf = torch.empty(7, dtype=torch.float64).pin_memory().numpy()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")     # > 50 MB L2 of the H100

    def barrier():
        if multi:
            dist.barrier()
        torch.cuda.synchronize()

    cx_phase_ms = {}

    def make_steps(cx, incremental=False):
        """The two step functions on context cx.  Streamed workload: the frame pushed is always the one the FIFO is about to
        drop (push number p re-pushes frame p % N_FRAMES, counted per context over ALL steps, warm-up included), so the
        map's content — and the step's work — stay constant."""
        pushes = [0]
        phase_ms = cx_phase_ms.setdefault(id(cx), [0.0, 0.0, 0.0, 0.0, 0])      # extract, odometry, push, rebuild, steps (event-timed)

        def step_resident(k):
            sw = sweeps[k % len(sweeps)]
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)] if stream_wl else None
            if ev: ev[0].record(stream)
            cx.extract_resident(sw["q"])
            if ev: ev[1].record(stream)
            pose, st, nds = cx.odometry_resident(sw["guess"], ITERS, mode=L.MODE_GN, want_stats=False)
            if stream_wl:
                ev[2].record(stream)
                fd = frames_dev[pushes[0] % N_FRAMES]
                pushes[0] += 1
                if incremental:     # SURVEY §8 (f2): push + incremental merge of the resident voxel entries (same resulting map)
                    ev[3].record(stream)
                    cx.map_update_device(fd.data_ptr(), fd.numel() // psz, ident)
                else:
                    cx.map_push_frame_device(fd.data_ptr(), fd.numel() // psz, ident)
                    ev[3].record(stream)
                    cx.map_rebuild()
                ev[4].record(stream); ev[4].synchronize()
                for i in range(4):
                    phase_ms[i] += ev[i].elapsed_time(ev[i + 1])
                phase_ms[4] += 1
            return pose, nds

        def step_e2e(k):
            i = k % len(sweeps)
            # Preprocessing node call: H2D raw sweep, D2H the three published clouds (pinned host buffers)
            surf, edge, cut = extract_host(cx, i, (out_surf, out_edge, out_cut))
            # LidarOdometry node call on the /surf_features cloud as received (host): H2D, D2H pose + surf_last_ds
            pose, st, ds = cx.odometry(surf, sweeps[i]["guess"], ITERS, mode=L.MODE_GN, ds_out=out_ds, pose_out=pose_buf, want_stats=False)
            h2d = len(pin_sweeps[i]) * psz + len(surf) * psz + 56
            d2h = (len(surf) + len(edge) + len(cut)) * psz + len(ds) * psz + 56
            if stream_wl:
                h2d += push_host()
            return pose, h2d, d2h, (surf, edge, cut, ds)

        def push_host():
            """buildLocalMap's push with the frame arriving from the host, then the rebuild; returns the bytes uploaded."""
            fh = frames_host[pushes[0] % N_FRAMES]
            pushes[0] += 1
            cx.map_push_frame(fh, ident)
            cx.map_rebuild()
            return len(fh) * psz + 56
        return step_resident, step_e2e, push_host

    step_resident, step_e2e, push_host_main = make_steps(ctx)

    def e2e_two_nodes(n_steps, n_warm):
        """The reference runs Preprocessing and LidarOdometry as two concurrent single-threaded nodes; so does this
        leg: one host thread + context + CUDA stream per node, the /surf_features hop through pinned host memory.
        A 256 MB L2-evicting write is issued per scan on a third stream INSIDE the timed region; in a pipelined steady
        state there is no gap "between" scans to put it in, so it runs under the scan's own kernels (conservative:
        it evicts the map continuously and competes for HBM bandwidth)."""
        ctx_pre = L.Context(prm, device=local_rank)
        s_pre = torch.cuda.Stream(); ctx_pre.set_stream(s_pre.cuda_stream)
        s_flush = torch.cuda.Stream()
        # The LidarOdometry stream gets the higher priority: its cooperative GN kernel needs every CTA resident and meets
        # at 10 grid barriers, so queueing behind the other node's CTAs (or the flush) costs it far more than it costs them.
        s_lo = torch.cuda.Stream(priority=-1)
        ctx.set_stream(s_lo.cuda_stream)
        nbuf = 3
        sets = [[torch.empty(cap * psz, dtype=torch.uint8).pin_memory().numpy().view(PT) for _ in range(3)] for _ in range(nbuf)]
        ev0 = torch.cuda.Event(enable_timing=True); ev1 = torch.cuda.Event(enable_timing=True)
        result = {}

        def stage_a(k, b):
            i = k % len(sweeps)
            with torch.cuda.stream(s_flush):
                flush.fill_(k & 0xff)
            surf, edge, cut = extract_host(ctx_pre, i, tuple(sets[b]))
            return (len(surf), len(edge), len(cut))

        def stage_b(k, b, item):
            ns, ne, nc = item
            i = k % len(sweeps)
            pose, st, ds = ctx.odometry(sets[b][0][:ns], sweeps[i]["guess"], ITERS, mode=L.MODE_GN, ds_out=out_ds, pose_out=pose_buf, want_stats=False)
            h2d = len(pin_sweeps[i]) * psz + ns * psz + 56
            if stream_wl:                      # the LidarOdometry node also maintains the map (buildLocalMap), after the scan
                h2d += push_host_main()
            result.update(pose=np.array(pose), h2d=h2d, d2h=(ns + ne + nc) * psz + len(ds) * psz + 56)

        barrier()
        try:
            run_two_stage_pipeline(n_warm + n_steps, n_warm, nbuf, stage_a, stage_b,
                                   on_start=lambda: ev0.record(s_pre), on_end=lambda: ev1.record(s_lo))
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1)
        finally:                 # also after a failure: every rank meets the barrier, the contexts go back to where they were
            barrier()
            ctx_pre.close()
            ctx.set_stream(stream.cuda_stream)
        return ms, (result["pose"], result["h2d"], result["d2h"])

    step_dist = {}                  # per-step device times of the last timed() call per step function (this rank)

    def timed(fn, n_steps, n_warm, prep=None, after_warmup=None, collective=True):
        """n_warm untimed steps, then n_steps steps each bracketed by its own CUDA-event pair on the launch stream, a 256 MB
        L2-evicting write between them.  Returns (this rank's total ms, last result)."""
        for k in range(n_warm):
            if prep: prep(k)
            fn(k)
        if after_warmup: after_warmup()
        if collective: barrier()
        else: torch.cuda.synchronize()
        tot_ms = 0.0
        last = None
        per_step = []
        with torch.cuda.stream(stream):
            for k in range(n_steps):
                if prep: prep(k)
                flush.fill_(k & 0xff)                       # evict L2 between steps (cold-cache scans)
                e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                last = fn(k)
                e1.record(stream)
                e1.synchronize()
                per_step.append(e0.elapsed_time(e1))
                tot_ms += per_step[-1]
        if collective: barrier()
        else: torch.cuda.synchronize()
        step_dist[fn.__name__] = per_step
        return tot_ms, last

    def over_ranks(ms):
        """(max over ranks, per-rank list) of a rank-local time."""
        if not multi:
            return ms, [ms]
        t = torch.tensor([ms], dtype=torch.float64, device="cuda")
        allt = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(allt, t)
        per = [float(x.item()) for x in allt]
        return max(per), per

    def prep_for(cx):
        def prep(k):
            cx.upload_scan(sweeps[k % len(sweeps)]["pts"])     # untimed: the sweep is resident when the step starts
        return prep

    # ---- timed region 1: device-resident; counters cover exactly the timed steps
    cnt_box = {}
    with clk:
        def after_warm():
            ctx.counters(reset=True)
            for v in cx_phase_ms.values():
                v[:] = [0.0, 0.0, 0.0, 0.0, 0]
        ms_res_local, last = timed(step_resident, steps, warmup, prep_for(ctx), after_warmup=after_warm)
        phases_main = list(cx_phase_ms.get(id(ctx), [0, 0, 0, 0, 0]))
        cnt = ctx.counters(reset=True)
        # C-bar of the LAST timed scan's queries at its start pose, while they are still resident (the later legs replace them)
        blk = ctx.knn_block_stats(sweeps[(steps - 1) % len(sweeps)]["guess"])
        ms_res, ms_res_ranks = over_ranks(ms_res_local)
        # ---- timed region 2: end to end with host buffers
        ms_seq_local, last_seq = timed(step_e2e, steps, warmup)
        ms_seq, _ = over_ranks(ms_seq_local)
        # copies: the later legs reuse the pinned output buffers the last e2e step's clouds are views of
        e2e_out = {"e2e_pose": np.array(last_seq[0], np.float64)}
        for name, cloud in zip(("e2e_surf", "e2e_edge", "e2e_cutted", "e2e_surf_ds"), last_seq[3]):
            e2e_out[name] = np.ascontiguousarray(cloud).view(np.float32).reshape(len(cloud), psz // 4).copy()
        # Sharded runs keep the one-thread e2e leg.  The two-node leg put each rank's GN exchange (a kernel that waits for its
        # peers) next to a second host thread and context on the same GPU; it ran on 2 GPUs, but on 8 every rank's exchange
        # hit its 6 s wait bound — not understood yet, so not shipped.
        two_node_error = None
        if args.e2e == "sequential" or sharded:
            ms_e2e, last_e2e = ms_seq, last_seq
        else:
            ms_e2e, last_e2e, two_node_error = resolve_e2e(lambda: e2e_two_nodes(steps, warmup), over_ranks, ms_seq, last_seq)
    clocks = clk.summary()
    ctx.counters(reset=True)

    def dist_of(name):
        v = sorted(step_dist.get(name) or [])
        return {"min": v[0], "median": v[len(v) // 2], "max": v[-1]} if v else None
    step_ms = {"resident": dist_of("step_resident"), "e2e_sequential": dist_of("step_e2e")}

    replicas = multi and not sharded
    scans_total = steps * (world if replicas else 1)
    value = scans_total / (ms_res * 1e-3)
    e2e_val = scans_total / (ms_e2e * 1e-3)

    # ---- roofline of the kNN+Jacobian kernel (algorithmic bytes per SURVEY.md §8 d)
    peak, peak_src = measured_peak()

    def roofline_from(cn, blk27):
        if not cn.knn_launches:
            return None
        nq, c27 = blk27                                       # resident queries of the last scan, at its start pose
        cbar27 = c27 / max(nq, 1)
        qpl = cn.knn_queries / cn.knn_launches                # device-side count: queries searched per pass
        cex = cn.knn_candidates / max(cn.knn_queries, 1)      # candidates examined per query after pruning
        t_launch = cn.knn_ms * 1e-3 / cn.knn_launches
        b8d = qpl * (16 + 27 * 8 + 16 * cbar27)
        bex = qpl * (16 + 27 * 8 + 16 * cex)
        return {"queries_per_launch": qpl, "candidates_per_query": cbar27, "examined_per_query": cex,
                "algorithmic_bytes_per_launch": b8d, "us_per_launch": t_launch * 1e6, "achieved": b8d / t_launch / 1e9,
                "frac": b8d / t_launch / 1e9 / peak,
                "examined": {"bytes_per_launch": bex, "achieved": bex / t_launch / 1e9, "frac": bex / t_launch / 1e9 / peak},
                "min_bytes_per_launch": qpl * 96.0, "passes_timed": int(cn.knn_launches),
                "timing": "CUDA-event pair around the kernel on the launch stream, inside the timed region"}

    roof = roofline_from(cnt, blk)
    if roof is not None:
        roof["timing"] += f", on every {KTIME_EVERY}th scan (the other scans run without the pair: it costs the step ~8-10 us)"
        traffic, traffic_src = None, None
        tp = os.path.join(ROOT, "profiles", "knn_traffic.json")
        if os.path.exists(tp):
            try:
                tj = json.load(open(tp))
                traffic, traffic_src = tj.get("dram_bytes_per_launch"), tj.get("source")
            except Exception:
                pass
        roof = {"bound": "hbm", "kernel": "k_gn_persistent / k_knn_plane (one GN pass of the kNN+plane+Jacobian+reduce+solve kernel body)",
                "unit": "GB/s", "peak": peak, "peak_source": peak_src, "traffic": traffic, "traffic_source": traffic_src,
                "accounting": "achieved = SURVEY §8(d) bytes (16 + 27*8 + 16*C-bar per query, C-bar = points in the query's 27 cells, "
                              "queries counted on the device) / CUDA-event time of one pass over the timed steps; `examined` = the same with the "
                              "candidates the pruned search actually fetched",
                **roof}

    # ---- the same kernel where it is less latency-bound (N = 1, default workload only; never allowed to break the bench line):
    # (a) every surf feature of the 24k sweep a query (leaf_scan = 0) against the 1 M-pt map,
    # (b) every return of a 130k-pt HDL-64E sweep a query against a 10 M-pt (HBM-resident) map, one thread per query.
    if roof is not None and not multi and kind == "horizon" and not args.dense_queries and not args.no_dense_probe:
        probes = {}
        try:
            dprm = L.default_params(0); dprm.leaf_scan = 0.0
            dctx = L.Context(dprm, device=local_rank)
            dctx.set_stream(stream.cuda_stream)
            dctx.map_set_points(m)
            dctx.set_kernel_timing(True)
            with torch.cuda.stream(stream):
                for k in range(24):
                    sw = sweeps[k % len(sweeps)]
                    dctx.upload_scan(sw["pts"])
                    flush.fill_(k & 0xff)
                    dctx.extract_resident(sw["q"])
                    dctx.odometry_resident(sw["guess"], ITERS, mode=L.MODE_GN, want_stats=False)
                    if k == 3:
                        dctx.counters(reset=True)
            r = roofline_from(dctx.counters(), dctx.knn_block_stats(sweeps[23 % len(sweeps)]["guess"]))
            dctx.close()
            if r:
                probes["surf_24k_vs_1M"] = {"what": "every surf feature of the 24k sweep a query (leaf_scan = 0), 1 M-pt map, 20 scans", **r}
        except Exception as e:      # noqa: BLE001
            probes["surf_24k_vs_1M"] = {"error": str(e)[:200]}
        try:
            from liliom_b200 import synth
            big, _ = synth.make_map(10_000_000)
            T = synth.default_true_pose()
            hdl, _q = synth.make_hdl64_sweep(T)
            feats = np.ones((len(hdl), 4), np.float32)
            feats[:, 0] = hdl["x"]; feats[:, 1] = hdl["y"]; feats[:, 2] = hdl["z"]
            bctx = L.Context(L.default_params(0), device=local_rank)
            bctx.set_stream(stream.cuda_stream)
            bctx.map_set_points(big)
            del big
            bctx.upload_feats(feats)
            bctx.set_kernel_timing(True)
            g = synth.perturbed_pose(T)
            with torch.cuda.stream(stream):
                for k in range(8):
                    flush.fill_(k & 0xff)
                    pz, _ = bctx.scan_to_map_resident(g, ITERS, mode=L.MODE_GN)
                    if k == 2:
                        bctx.counters(reset=True)
            r = roofline_from(bctx.counters(), bctx.knn_block_stats(g))
            bctx.close()
            if r:
                probes["hdl_130k_vs_10M"] = {"what": "every return of a 130k-pt HDL-64E sweep a query, 10 M-pt map (HBM-resident), 5 scans x 10 passes",
                                             "pose_err_m": float(np.linalg.norm(pz[4:] - T[4:])), **r}
        except Exception as e:      # noqa: BLE001
            probes["hdl_130k_vs_10M"] = {"error": str(e)[:200]}
        roof["dense_probe"] = probes

    def incremental_leg(k1, pose_ref):
        """The streamed workload on ONE GPU with liliom_map_update (SURVEY §8 f2) in place of push_frame + rebuild: same map, same poses."""
        try:
            c2 = new_context(False)
            install_map(c2)
            s2_res, _, _ = make_steps(c2, incremental=True)
            ms2, last2 = timed(s2_res, k1, 3, prep_for(c2), after_warmup=lambda: cx_phase_ms[id(c2)].__setitem__(slice(None), [0.0, 0.0, 0.0, 0.0, 0]),
                               collective=False)
            ph2 = cx_phase_ms.get(id(c2), [0, 0, 0, 0, 0])
            c2.close()
            return {"value": k1 / (ms2 * 1e-3), "unit": "scans/s", "ms_per_step": ms2 / k1, "steps": k1,
                    "map_update_ms": (ph2[3] / ph2[4]) if ph2[4] else None,
                    "pose_max_abs_diff_vs_rebuild": float(np.abs(np.asarray(last2[0]) - np.asarray(pose_ref)).max()),
                    "what": "liliom_map_update (incremental merge of the resident voxel entries) instead of push_frame + rebuild"}
        except Exception as e:      # noqa: BLE001
            return {"error": str(e)[:200]}

    inc_single = None
    if stream_wl and not multi and not args.no_extra_legs:
        inc_single = incremental_leg(steps, last[0])

    # ---- N > 1, sharded: the SAME workload on one GPU (rank 0, fewer steps), and the replicas number as a secondary key
    same1, repl = None, None
    if sharded and not args.no_extra_legs:
        if rank == 0:
            try:
                c1 = new_context(False)
                install_map(c1)
                s1_res, _, _ = make_steps(c1)
                k1 = max(3, min(steps, 20))
                ms1, last1 = timed(s1_res, k1, 3, prep_for(c1), after_warmup=lambda: cx_phase_ms[id(c1)].__setitem__(slice(None), [0.0, 0.0, 0.0, 0.0, 0]),
                                   collective=False)
                ph1 = cx_phase_ms.get(id(c1), [0, 0, 0, 0, 0])
                c1.close()
                inc1 = incremental_leg(k1, last1[0])
                same1 = {"value": k1 / (ms1 * 1e-3), "unit": "scans/s", "ms_per_step": ms1 / k1, "steps": k1, "incremental_map": inc1,
                         "step_breakdown_ms": ({k: ph1[i] / ph1[4] for i, k in enumerate(("extract", "scan_vg_and_gn", "push_frame", "map_rebuild"))}
                                               if ph1[4] else None),
                         "pose_max_abs_diff_vs_sharded": float(np.abs(np.asarray(last1[0]) - np.asarray(last[0])).max())
                         if (k1 - 1) % len(sweeps) == (steps - 1) % len(sweeps) else None,
                         "what": "the same streamed workload (full map, no sharding) on ONE GPU, measured by rank 0 in this run"}
            except Exception as e:      # noqa: BLE001
                same1 = {"error": str(e)[:200]}
        barrier()
        try:
            from liliom_b200 import synth
            rprm = L.default_params(0)
            rc = L.Context(rprm, device=local_rank)
            rc.set_stream(stream.cuda_stream)
            m1, _ = synth.make_map(1_000_000)
            rc.map_set_points(m1)
            T0 = synth.default_true_pose()
            rs = []
            for k in range(4):
                T = np.array(T0); T[4] += 0.7 * (k + rank); T[5] += 0.15 * (k + rank)
                p_, q_ = synth.make_horizon_sweep(T, seed=1 + k + rank)
                rs.append((p_, q_, synth.perturbed_pose(T)))

            def rstep(k):
                p_, q_, g_ = rs[k % len(rs)]
                rc.extract_resident(q_)
                return rc.odometry_resident(g_, ITERS, mode=L.MODE_GN, want_stats=False)

            def rprep(k):
                rc.upload_scan(rs[k % len(rs)][0])
            kr = max(10, min(steps, 100))
            msr_local, _ = timed(rstep, kr, 5, rprep)
            msr, msr_ranks = over_ranks(msr_local)
            rc.close()
            repl = {"value": kr * world / (msr * 1e-3), "unit": "scans/s", "steps": kr, "ms_per_step_ranks": [x / kr for x in msr_ranks],
                    "what": "independent scan streams, one per GPU, each the N = 1 workload (24k-pt Horizon sweep vs 1 M-pt map): weak scaling, no collective"}
        except Exception as e:      # noqa: BLE001
            repl = {"error": str(e)[:200]}

    if rank != 0:
        ctx.close()
        return None
    cpu = None if (args.no_cpu_baseline or multi) else cpu_baseline_leg(kind, m, sweeps[:4])
    pose, nq = last
    per_rank = [x / steps for x in ms_res_ranks]
    cfg = config_dict(kind, len(sweeps[0]["pts"]), n_map, world, args.multi)
    run = {"queries_per_scan": int(nq), "dense_queries": bool(args.dense_queries), "map_points_installed": int(n_map_installed),
                "exchange": (None if not sharded else "29 fp64 sums per GN iteration: " +
                             ("ncclAllReduce + update kernel per iteration" if use_nccl_exchange else
                              "fused into the persistent GN kernel over NVLink peer memory (one launch per scan and rank)") +
                             "; map maintenance: one 2-scalar ncclAllReduce per rebuild (map-size guard)")}
    line = {
        "metric": METRIC, "value": value, "unit": "scans/s", "n_gpus": world, "steps": steps, "warmup": warmup,
        "ms_per_step": ms_res / steps, "higher_is_better": True,
        "scaling": "strong" if sharded else "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": cfg, "run": run,
        "step_ms": step_ms, "gpu_launches": int(cnt.launches),
        "lib_calls": int(cnt.lib_launches),
        "e2e": {"value": e2e_val, "unit": "scans/s", "ms_per_step": ms_e2e / steps,
                "h2d_bytes_per_step": int(last_e2e[1]), "d2h_bytes_per_step": int(last_e2e[2]),
                "mode": ("sequential: one host thread calls the Preprocessing-node entry point, the LidarOdometry-node entry point"
                         + (" and the map maintenance" if stream_wl else "") + " in turn"
                         + ("" if not two_node_error else " (the two-node leg failed and is not reported: " + two_node_error + ")")
                         if (args.e2e == "sequential" or sharded or two_node_error) else
                         "two-nodes: Preprocessing and LidarOdometry contexts on two host threads / CUDA streams" + (" per rank" if multi else "") +
                         ", as the reference's two ROS nodes" + (" (the LidarOdometry thread also pushes the frame and rebuilds the map)" if stream_wl else "") +
                         "; /surf_features hop through pinned host memory; one 256 MB L2-evicting write per scan on a third stream inside "
                         "the timed region (sequential_value: one thread, flush strictly between scans — the like-for-like figure against "
                         "the strictly sequential reference arm)"),
                "sequential_value": scans_total / (ms_seq * 1e-3), "sequential_ms_per_step": ms_seq / steps},
        "clocks": clocks,
        "roofline": roof,
        "cpu_baseline": cpu,
        "pose_err_m": float(np.linalg.norm(np.asarray(pose)[4:] - sweeps[(steps - 1) % len(sweeps)]["T"][4:])),
        "host": {"cpus": os.cpu_count(), "cpus_usable": len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else None,
                 "affinity": os.environ.get("LILIOM_BENCH_AFFINITY"),
                 "note": "one python process per GPU; every library call ends in a stream synchronise on the host"},
    }
    if inc_single is not None:
        line["incremental_map"] = inc_single
    if stream_wl and phases_main[4]:
        line["step_breakdown_ms"] = {k: phases_main[i] / phases_main[4] for i, k in enumerate(("extract", "scan_vg_and_gn", "push_frame", "map_rebuild"))}
    if multi:
        line["ms_per_step_ranks"] = {"min": min(per_rank), "median": float(np.median(per_rank)), "max": max(per_rank), "all": per_rank}
    if sharded:
        line["same_workload_1gpu"] = same1
        line["replicas"] = repl
        if same1 and "value" in same1:
            line["speedup_vs_1gpu_same_workload"] = value / same1["value"]
    if fallback_note or exchange_note:
        line["note"] = "; ".join(x for x in (fallback_note, exchange_note) if x)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {"resident_pose": np.array(pose, np.float64), "resident_n_queries": np.array([nq], np.float64),
                                         **e2e_out})
    print(json.dumps(line), flush=True)
    ctx.close()
    return None


if __name__ == "__main__":
    main()
