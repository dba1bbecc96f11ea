#!/usr/bin/env python
"""Local-map maintenance of several odometry sessions on one GPU.  Workload per session: the headline Horizon step (a seeded
24k-point sweep extracted on the device, 10 GN iterations) against the session's OWN local map, a full 20-frame FIFO of its
last down-sampled scans (steady state: every update pops a frame), not an installed static map.

Map update alone, timed per step for all B sessions (the scan and the odometry call in front of it are not timed):
  (h) B solo liliom_map_update calls on the host copy of each scan (what a caller had to write before
      liliom_map_update_resident: the cloud downloaded through ds_out, uploaded again; the upload is in the time, the download
      is part of the odometry call and is not);
  (i) B solo liliom_map_update_resident calls;
  (j) one liliom_map_update_batch call.
The three legs leave identical maps, so they alternate step by step on the same sessions.
Whole fleet step (per-session upload of the raw sweep, liliom_extract_resident_batch, map update with the previous scan's frame
and pose, liliom_odometry_resident_batch_ex), timed end to end, in alternating blocks:
  (H) map update by B solo liliom_map_update calls, the odometry batch downloading every ds_out;
  (J) map update by one liliom_map_update_batch, no cloud crossing PCIe.
Both legs push the same frames under the same poses (the last scan of a (J) block is downloaded, untimed, before an (H) block
starts), so the sessions' maps do not depend on the order of the blocks.
Every row is measured --runs times; each figure is the median over a run's steps, printed as the median over the runs with the
smallest and largest run beside it (the run-to-run spread).  Prints the card, its power limit and maximum SM clock first.  Reads
device state only.
usage: map_batch_bench.py [--sessions 1 2 4 8 16 32] [--steps 30] [--warmup 5] [--runs 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import liliom_b200 as L  # noqa: E402
from liliom_b200 import synth  # noqa: E402

ITERS = 10
FIFO = 20
DS_CAP = 32768


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def spread(runs):
    """median over the runs, and (smallest, largest) run"""
    return [round(float(np.median(runs)), 4), round(float(min(runs)), 4), round(float(max(runs)), 4)]


class Fleet:
    def __init__(self, B, sweeps):
        self.B, self.sweeps = B, sweeps
        self.ctxs = [L.Context(variant=0) for _ in range(B)]
        self.ds = [np.zeros(DS_CAP, c.dtype) for c in self.ctxs]          # host copies of surf_last_ds, allocated once
        self.nds = np.zeros(B, np.int32)
        self.poses = np.zeros((B, 7))
        self.k = 0
        lib, ip = L._binding.lib(), C.POINTER(C.c_int)
        self.lib = lib
        self.handles = (C.c_void_p * B)(*[c._h for c in self.ctxs])
        self.outs = (C.c_void_p * B)(*[d.ctypes.data for d in self.ds])
        self.cnt, self.mni = np.full(B, ITERS, np.int32), np.full(B, 15, np.int32)
        self.caps, self.status = np.full(B, DS_CAP, np.int32), np.zeros(B, np.int32)
        self._ip = lambda a: a.ctypes.data_as(ip)

    def sweep(self, s):
        return self.sweeps[(self.k + s) % len(self.sweeps)]

    def odo_solo(self, s):
        """scan + solo odometry of session s, its DS cloud downloaded: the step in front of a map update"""
        c, sw = self.ctxs[s], self.sweep(s)
        c.upload_scan(sw["pts"])
        c.extract_resident(sw["q"])
        pose = np.array(sw["guess"], dtype=np.float64)
        n = C.c_int()
        rc = self.lib.liliom_odometry_resident(c._h, pose.ctypes.data_as(C.POINTER(C.c_double)), ITERS, 15, L.MODE_GN, None,
                                               self.ds[s].ctypes.data_as(C.c_void_p), DS_CAP, C.byref(n))
        self.nds[s] = n.value
        self.poses[s] = pose if rc == 0 else sw["T"]                      # no map yet: the frame goes in under its true pose

    def odo_batch(self, download):
        dp = C.POINTER(C.c_double)
        poses = np.array([self.sweep(s)["guess"] for s in range(self.B)])
        rc = self.lib.liliom_odometry_resident_batch_ex(self.handles, self.B, poses.ctypes.data_as(dp), self._ip(self.cnt), self._ip(self.mni),
                                                        L.MODE_GN, None, self.outs if download else None, self._ip(self.caps),
                                                        self._ip(self.nds) if download else None, self._ip(self.status))
        assert rc == 0 and not self.status.any(), (rc, self.status)
        self.poses = poses

    def update(self, leg):
        if leg == "h":
            for s, c in enumerate(self.ctxs):
                c.map_update(self.ds[s][:self.nds[s]], self.poses[s])
        elif leg == "i":
            for s, c in enumerate(self.ctxs):
                c.map_update_resident(self.poses[s])
        else:
            _, status = L.map_update_batch(self.ctxs, self.poses)
            assert not status.any(), status

    def fill(self):
        for _ in range(FIFO + 2):
            for s in range(self.B):
                self.odo_solo(s)
            self.update("i")
            self.k += 1

    def map_only(self, steps):
        """`steps` samples (ms for all B sessions) per leg, the legs alternating step by step"""
        lat = {"h": [], "i": [], "j": []}
        for n in range(3 * steps):
            leg = "hij"[n % 3]
            for s in range(self.B):
                self.odo_solo(s)
            torch.cuda.synchronize()
            t = time.perf_counter()
            self.update(leg)
            lat[leg].append((time.perf_counter() - t) * 1e3)
            self.k += 1
        return lat

    def fleet_steps(self, leg, steps):
        """`steps` whole fleet steps with the map update of `leg`; returns their times in ms"""
        lat = []
        for _ in range(steps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            for s, c in enumerate(self.ctxs):
                c.upload_scan(self.sweep(s)["pts"])
            _, st = L.extract_resident_batch(self.ctxs, np.array([self.sweep(s)["q"] for s in range(self.B)]))
            self.update(leg)
            self.odo_batch(download=leg == "h")
            lat.append((time.perf_counter() - t) * 1e3)
            assert not st.any(), st
            self.k += 1
        return lat

    def close(self):
        for c in self.ctxs:
            c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, nargs="*", default=[1, 2, 4, 8, 16, 32])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("map_batch_bench.py measures on a CUDA device; none is visible")
    print(json.dumps(dict(card(), iters=ITERS, fifo=FIFO, steps=args.steps, runs=args.runs, figures="[median of runs, min run, max run], ms")),
          flush=True)
    T0 = synth.default_true_pose()
    sweeps = []
    for k in range(8):
        T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        sweeps.append(dict(T=T, guess=synth.perturbed_pose(T), pts=pts, q=q))
    for B in args.sessions:
        f = Fleet(B, sweeps)
        f.fill()
        row = dict(sessions=B, map_points=int(np.median([c.map_size() for c in f.ctxs])), ds_points=int(np.median(f.nds)))
        f.map_only(args.warmup)
        runs = [f.map_only(args.steps) for _ in range(args.runs)]
        for leg, name in (("h", "h_host_update"), ("i", "i_resident_update"), ("j", "j_batch_update")):
            row[f"{name}_ms"] = spread([np.median(r[leg]) for r in runs])
        def block(leg, n):
            if leg == "h":      # a (J) block downloads nothing: the scan in front of an (H) block is stepped again with its
                f.odo_batch(download=True)      # download (not timed), so that (H) pushes the frame (J) would, and the maps stay equal
            return f.fleet_steps(leg, n)
        for leg in "hj":
            block(leg, args.warmup)
        steps = {"h": [], "j": []}
        for _ in range(args.runs):
            for leg in "hj":
                steps[leg].append(np.median(block(leg, args.steps)))
        row["H_fleet_step_host_maps_ms"] = spread(steps["h"])
        row["J_fleet_step_batch_maps_ms"] = spread(steps["j"])
        print(json.dumps(row), flush=True)
        f.close()


if __name__ == "__main__":
    main()
