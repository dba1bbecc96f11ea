#!/usr/bin/env python
"""The fleet's front door: getting B sessions' sweeps onto the device, three ways, and the whole fleet step behind two of them.
Per session: --variant horizon, a seeded Horizon sweep as Livox CustomPoint records (stride 20, 20 B per point) or as PCL
points (48 B); --variant rot, a seeded 130k-point HDL-64E sweep as a packed Velodyne PointCloud2 (22 B per point) or as PCL
points (32 B).
  (a) B liliom_upload_scan calls of the PCL points (each synchronises);
  (b) B solo converts (liliom_convert_livox / liliom_convert_pc2, each synchronises);
  (c) one liliom_convert_batch;
  (fa) / (fc) the whole fleet step with (a) / (c) in front of one liliom_extract_resident_batch, one
  liliom_odometry_resident_batch_ex (GN, 4 iterations) and one liliom_map_update_batch.
Each leg runs with its payloads in pageable memory and in page-locked memory (torch pin_memory).  The legs alternate inside
every run; a run times --steps calls of each leg after --warmup, and the row reports the median of --runs runs with the smallest
and largest run.  Prints the card, its power limit and maximum SM clock, then one JSON line per (variant, memory, B).
usage: wire_batch_bench.py [--variant {horizon,rot} ...] [--sessions 1 2 4 8 16 32] [--steps 20] [--warmup 3] [--runs 3]
                           [--out FILE]"""
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

IP = C.POINTER(C.c_int)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def placed(a: np.ndarray, pinned: bool) -> np.ndarray:
    """a's bytes in pageable memory (a copy) or in page-locked memory (a torch pin_memory buffer), same dtype and shape."""
    raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    if pinned:
        t = torch.empty(raw.size, dtype=torch.uint8, pin_memory=True)
        buf = t.numpy()
        buf[:] = raw
        placed.keep.append(t)
    else:
        buf = raw.copy()
    return buf.view(a.dtype).reshape(a.shape)


placed.keep = []


def livox_records(pts, t_end=100_000_000):
    """A Horizon sweep (PT48, intensity = line + 0.1 * relative time) as Livox CustomPoint records in time order."""
    pts = pts[np.isfinite(pts["intensity"]) & (pts["intensity"] >= 0) & (pts["intensity"] < 6)]
    frac = (pts["intensity"] - np.floor(pts["intensity"])).astype(np.float64)
    order = np.argsort(frac, kind="stable")
    pts, frac = pts[order], frac[order]
    r = np.zeros(len(pts), L.LIVOX20)
    off = np.minimum(np.round(frac / 0.1 * t_end), t_end).astype(np.uint32)
    off[-1] = t_end
    r["offset_time"] = off
    r["x"], r["y"], r["z"] = pts["x"], pts["y"], pts["z"]
    r["reflectivity"] = 50
    r["line"] = np.floor(pts["intensity"]).astype(np.uint8)
    return r


class Fleet:
    """B sessions of one variant with their payloads placed in one kind of memory, and the prebuilt arguments of every call."""

    def __init__(self, variant, B, sweeps, m, pinned):
        self.B, self.rot = B, variant == "rot"
        self.cs = [L.Context(variant=1 if self.rot else 0) for _ in range(B)]
        for c in self.cs:
            c.map_set_points(m)
        self.lib = L._binding.lib()
        self.h = (C.c_void_p * B)(*[c._h for c in self.cs])
        self.pcl, self.wire, keep = [], (L.WireMsg * B)(), []
        for i in range(B):
            s = sweeps[i % len(sweeps)]
            self.pcl.append(placed(s["pcl"], pinned))
            if self.rot:
                msg = s["pc2"]
                data = placed(msg.data, pinned)
                cm, f = L.PC2(data, msg.height, msg.width, msg.point_step, msg.row_step, msg.fields).c_msg()
                keep += [data, cm, f]
                self.wire[i].kind, self.wire[i].pc2 = L.WIRE_PC2, C.pointer(cm)
            else:
                rec = placed(s["livox"], pinned)
                keep.append(rec)
                self.wire[i].kind, self.wire[i].custom_pts, self.wire[i].n, self.wire[i].stride = L.WIRE_LIVOX, rec.ctypes.data, len(rec), 20
        self.keep = keep
        self.q = np.ascontiguousarray(np.stack([sweeps[i % len(sweeps)]["q"] for i in range(B)]), np.float64)
        self.qlb = np.ascontiguousarray(np.tile([1.0, 0.0, 0.0, 0.0], (B, 1)), np.float64)
        self.guess = np.ascontiguousarray(np.tile(synth.perturbed_pose(synth.default_true_pose()), (B, 1)), np.float64)
        self.n = np.zeros(B, np.int32)
        self.st = np.zeros(B, np.int32)
        self.cnt = np.zeros((3, B), np.int32)
        self.mc = np.full(B, 4, np.int32)
        self.mni = np.full(B, 15, np.int32)
        self.nmap = np.zeros(B, np.int32)

    def upload(self):
        for c, p in zip(self.cs, self.pcl):
            assert self.lib.liliom_upload_scan(c._h, p.ctypes.data, len(p)) == 0

    def solo(self):
        n = C.c_int()
        for i, c in enumerate(self.cs):
            w = self.wire[i]
            rc = (self.lib.liliom_convert_pc2(c._h, w.pc2, None, 0, C.byref(n)) if self.rot else
                  self.lib.liliom_convert_livox(c._h, w.custom_pts, w.n, w.stride, None, 0))
            assert rc == 0

    def batch(self):
        assert self.lib.liliom_convert_batch(self.h, self.B, self.wire, None, None, self.n.ctypes.data_as(IP), self.st.ctypes.data_as(IP)) == 0
        assert (self.st == 0).all()

    def step(self, ingest):
        ingest()
        dp = C.POINTER(C.c_double)
        assert self.lib.liliom_extract_resident_batch(self.h, self.B, self.q.ctypes.data_as(dp), self.qlb.ctypes.data_as(dp),
                                                      *[self.cnt[k].ctypes.data_as(IP) for k in range(3)], self.st.ctypes.data_as(IP)) == 0
        poses = self.guess.copy()
        assert self.lib.liliom_odometry_resident_batch_ex(self.h, self.B, poses.ctypes.data_as(dp), self.mc.ctypes.data_as(IP),
                                                          self.mni.ctypes.data_as(IP), L.MODE_GN, None, None, None, None,
                                                          self.st.ctypes.data_as(IP)) == 0
        assert self.lib.liliom_map_update_batch(self.h, self.B, poses.ctypes.data_as(dp), self.nmap.ctypes.data_as(IP),
                                                self.st.ctypes.data_as(IP)) == 0

    def close(self):
        for c in self.cs:
            c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", nargs="*", choices=("horizon", "rot"), default=["horizon", "rot"])
    ap.add_argument("--sessions", type=int, nargs="*", default=[1, 2, 4, 8, 16, 32])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wire_batch_bench.py measures on a CUDA device; none is visible")
    info = card()
    print(json.dumps(info), flush=True)
    m, _ = synth.make_map(1_000_000)
    T = synth.default_true_pose()
    rows = []
    for variant in args.variant:
        sweeps = []
        for k in range(4):
            Tk = np.array(T); Tk[4] += 0.4 * k
            if variant == "rot":
                pts, q, ring, step = synth.make_hdl64_sweep(Tk, seed=40 + k, grid=True)
                sweeps.append(dict(pcl=pts, pc2=synth.encode_pc2(pts, ring, step, "velodyne22"), q=q))
            else:
                pts, q = synth.make_horizon_sweep(Tk, seed=40 + k)
                rec = livox_records(pts)
                sweeps.append(dict(pcl=L.Context(variant=0).convert_livox(rec), livox=rec, q=q))
        for B in args.sessions:
            for pinned in (False, True):
                f = Fleet(variant, B, sweeps, m, pinned)
                legs = {"a_upload": f.upload, "b_solo": f.solo, "c_batch": f.batch,
                        "fa_step_upload": lambda: f.step(f.upload), "fc_step_batch": lambda: f.step(f.batch)}
                runs = {k: [] for k in legs}
                for k, fn in legs.items():
                    for _ in range(args.warmup):
                        fn()
                for _ in range(args.runs):
                    for k, fn in legs.items():             # the legs alternate inside every run
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        for _ in range(args.steps):
                            fn()
                        torch.cuda.synchronize()
                        runs[k].append((time.perf_counter() - t0) / args.steps * 1e3)
                row = dict(variant=variant, memory="pinned" if pinned else "pageable", sessions=B,
                           bytes_per_point=(22 if variant == "rot" else 20), pcl_bytes_per_point=(32 if variant == "rot" else 48),
                           points_per_session=[int(s["pcl"].shape[0]) for s in sweeps][:min(B, 4)])
                for k, v in runs.items():
                    row[f"{k}_ms"] = [round(float(np.median(v)), 4), round(float(min(v)), 4), round(float(max(v)), 4)]
                rows.append(row)
                print(json.dumps(row), flush=True)
                f.close()
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=info, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
