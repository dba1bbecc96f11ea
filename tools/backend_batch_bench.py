#!/usr/bin/env python
"""The backend's sliding-window LiDAR calls of several sessions on one GPU.  Each session has its own seeded keyframe stream
(synth.make_keyframe_sequence) stored in its own context, and a 40-keyframe local map (solo liliom_bmap_build, built once, not
timed).  A fleet window step is, for every session, one search of a 3-keyframe window and 16 evaluations of its blocks (15 LM
iterations and the marginalisation, as tools/backend_bench.py models them):
  (a) B solo loops: liliom_backend_window_correspond, then 16 liliom_backend_window_blocks, per session;
  (b) one liliom_backend_window_correspond_batch, then 16 liliom_backend_window_blocks_batch.
Both legs call the C ABI with argument arrays built once, so that the time is the library's, not the Python wrappers'.
The legs alternate over --rounds rounds of --steps timed steps each (after --warmup untimed ones).  Per B: the median, smallest
and largest of the rounds' median ms per fleet window step, the waits per step (each call ends in one stream synchronise),
and whether (a) and (b) gave byte-identical counts and blocks.  Prints the card, its power limit and maximum SM clock first.
--loop measures a fleet loop-closure tick instead (DESIGN.md §5's loop-closure row per session): each session's store holds
synth.make_keyframe_sequence(41, revisit=1) (its own seed); the source is the revisit keyframe listed 2 deg / 0.5 m off, the target
the 41 history keyframes, at the reference's ICP settings (leaf 0.4, 30 m, 100 iterations, 1e-6, 1e-6):
  (a) B solo liliom_loop_align calls;
  (b) one liliom_loop_align_batch.
Reads device state only.
--handoff measures a fleet keyframe hand-off tick instead, the worst tick, when every session's keyframe falls due together: each
session extracts its own seeded sweep (Horizon: synth.make_horizon_sweep with backend variant 0; HDL-64E: synth.make_hdl64_sweep
with variant 1) before every tick, untimed, and hands its three resident clouds to its backend with publishCloudLast's
translation:
  (a) B x (liliom_undistort_resident + liliom_kf_add_resident);
  (b) one liliom_undistort_resident_batch + one liliom_kf_add_resident_batch.
Each leg stores into backends of its own, whose arenas are grown before the timed window (the whole run's keyframes stored once,
then liliom_kf_clear), so that no timed call reallocates.  Fleets: all Horizon, all HDL-64E, and mixed (alternating).  The legs'
ids and counts of every tick and every session's last stored clouds are checked byte-identical in the same run.  The waits per
tick (waits_by_design) are derived from the calls' structure, not counted in the run.
--localmap measures a fleet's backend local map instead: each session stores its own seeded 40-keyframe stream
(synth.make_keyframe_sequence: stride 48 with backend variant 0, stride 32 with variant 1), and every tick lists the 40 keyframes
with their poses nudged per tick:
  (a) B solo liliom_bmap_build calls;
  (b) one liliom_bmap_build_batch.
A second row per B times the whole backend keyframe step: (a) per session the solo local map, window search and 16 block
evaluations; (b) the three batched calls (liliom_bmap_build_batch, liliom_backend_window_correspond_batch, 16
liliom_backend_window_blocks_batch).  Fleets: all Horizon, all ROT, and mixed (alternating).  Each leg has contexts of its own;
the legs' counts, windows and blocks of the last tick of every round, and both layers of every session at the end, are checked
byte-identical in the same run.
usage: backend_batch_bench.py [--loop | --handoff | --localmap] [--sessions 1 2 4 8 16 32] [--steps 20] [--warmup 3] [--rounds 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NKF = 40           # keyframes in the local map
WIN = 3            # window keyframes
EVALS = 16         # blocks evaluations per window


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def spread(v):
    return [round(float(np.median(v)), 4), round(float(min(v)), 4), round(float(max(v)), 4)]


def stream(seed):
    from liliom_b200 import synth
    return synth.make_keyframe_sequence(NKF, stride=48, seed=seed)


def nudge(pose, k):
    from liliom_b200 import synth
    dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.1 * k))
    return np.concatenate([synth.qmul(pose[:4], dq), pose[4:] + 0.005 * k * np.array([1.0, -0.5, 0.25])])


class Session:
    def __init__(self, seq):
        import liliom_b200 as L
        self.bp = L.backend_default_params(0)
        self.c = L.Context(variant=0)
        for e, s, _ in seq:
            self.c.kf_add(self.bp, e, s, download=False)
        self.c.bmap_build(self.bp, list(range(NKF)), [p for _, _, p in seq])
        self.ids = np.arange(NKF - WIN, NKF, dtype=np.int32)
        self.poses_l = np.array([nudge(seq[i][2], 1) for i in self.ids])
        self.bodies = [np.array([nudge(p, 2 + j) for p in self.poses_l]) for j in range(EVALS)]
        # each leg's own results: counts, then the 16 blocks
        self.res = {leg: (np.zeros(WIN, np.int32), np.zeros(WIN, np.int32), [np.zeros((WIN, 2, 29)) for _ in range(EVALS)]) for leg in "ab"}


def ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Fleet:
    """B sessions and the C arguments of both legs, built once: the timed window holds the library's calls only."""

    def __init__(self, S):
        import liliom_b200 as L
        self.S, self.lib, B = S, L._binding.lib(), len(S)
        P, D = C.POINTER(C.c_int), C.POINTER(C.c_double)
        self.handles = (C.c_void_p * B)(*[s.c._h for s in S])
        self.bps = (L.BackendParams * B)(*[s.bp for s in S])
        self.ids = (P * B)(*[ptr(s.ids, C.c_int) for s in S])
        self.poses = (D * B)(*[ptr(s.poses_l, C.c_double) for s in S])
        self.k = np.full(B, WIN, np.int32)
        self.ne = (P * B)(*[ptr(s.res["b"][0], C.c_int) for s in S])
        self.ns = (P * B)(*[ptr(s.res["b"][1], C.c_int) for s in S])
        self.bodies = [(D * B)(*[ptr(s.bodies[j], C.c_double) for s in S]) for j in range(EVALS)]
        self.outs = [(D * B)(*[ptr(s.res["b"][2][j], C.c_double) for s in S]) for j in range(EVALS)]
        self.status = np.zeros(B, np.int32)

    def leg_a(self):
        for s in self.S:
            ne, ns, out = s.res["a"]
            rc = self.lib.liliom_backend_window_correspond(s.c._h, C.byref(s.bp), ptr(s.ids, C.c_int), ptr(s.poses_l, C.c_double), WIN,
                                                           ptr(ne, C.c_int), ptr(ns, C.c_int))
            assert rc == 0, rc
            for j in range(EVALS):
                rc = self.lib.liliom_backend_window_blocks(s.c._h, ptr(s.bodies[j], C.c_double), WIN, ptr(out[j], C.c_double))
                assert rc == 0, rc

    def leg_b(self):
        B, st = len(self.S), ptr(self.status, C.c_int)
        rc = self.lib.liliom_backend_window_correspond_batch(self.handles, B, self.bps, self.ids, self.poses, ptr(self.k, C.c_int),
                                                             self.ne, self.ns, st)
        assert rc == 0 and not self.status.any(), (rc, self.status)
        for j in range(EVALS):
            rc = self.lib.liliom_backend_window_blocks_batch(self.handles, B, self.bodies[j], ptr(self.k, C.c_int), self.outs[j], st)
            assert rc == 0 and not self.status.any(), (rc, self.status)

    def outputs(self, leg):
        """leg's results of every session as bytes; cleared for the next step"""
        out = b""
        for s in self.S:
            ne, ns, blocks = s.res[leg]
            out += ne.tobytes() + ns.tobytes() + b"".join(o.tobytes() for o in blocks)
            for a in [ne, ns] + blocks:
                a.fill(0)
        return out

    def prepare(self, leg):
        pass


LC_HIST = 41       # his_key_frames_ds at lc_map_width = 20
LC_LEAF = 0.4


def loop_stream(seed):
    from liliom_b200 import synth
    return synth.make_keyframe_sequence(LC_HIST, stride=48, seed=seed, revisit=1)


class LoopSession:
    def __init__(self, seq):
        import liliom_b200 as L
        from liliom_b200 import synth
        bp = L.backend_default_params(0)
        self.c = L.Context(variant=0)
        for e, s, _ in seq:
            self.c.kf_add(bp, e, s, download=False)
        p = seq[LC_HIST][2]
        qd = synth.q_from_axis_angle([0.1, -0.1, 1.0], np.deg2rad(2.0))
        self.src_ids = np.array([LC_HIST], np.int32)
        self.src_poses = np.concatenate([synth.qmul(qd, p[:4]), p[4:] + np.array([0.4, -0.25, 0.15])])
        self.tgt_ids = np.arange(LC_HIST, dtype=np.int32)
        self.tgt_poses = np.ascontiguousarray([q for _, _, q in seq[:LC_HIST]], np.float64).reshape(-1)
        self.res = {leg: L.LoopResult() for leg in "ab"}


class LoopFleet:
    """B sessions and the C arguments of both legs, built once."""

    def __init__(self, S):
        import liliom_b200 as L
        self.S, self.lib, B = S, L._binding.lib(), len(S)
        P, D = C.POINTER(C.c_int), C.POINTER(C.c_double)
        self.handles = (C.c_void_p * B)(*[s.c._h for s in S])
        self.si = (P * B)(*[ptr(s.src_ids, C.c_int) for s in S])
        self.sp = (D * B)(*[ptr(s.src_poses, C.c_double) for s in S])
        self.ti = (P * B)(*[ptr(s.tgt_ids, C.c_int) for s in S])
        self.tp = (D * B)(*[ptr(s.tgt_poses, C.c_double) for s in S])
        self.ks = np.ones(B, np.int32)
        self.kt = np.full(B, LC_HIST, np.int32)
        self.prm = (L.LoopParams * B)(*[L.LoopParams(LC_LEAF, 30.0, 100, 1e-6, 1e-6) for _ in S])
        self.out = (L.LoopResult * B)()
        self.status = np.zeros(B, np.int32)
        # leg (a)'s output pointers: the fields of each session's own LoopResult
        at = lambda r, name, t: C.cast(C.c_void_p(C.addressof(r) + getattr(L.LoopResult, name).offset), C.POINTER(t))   # noqa: E731
        self.solo_out = [(at(r, "T16", C.c_double), at(r, "fitness", C.c_double), at(r, "converged", C.c_int), at(r, "iters", C.c_int),
                          at(r, "n_src", C.c_int), at(r, "n_tgt", C.c_int)) for r in (s.res["a"] for s in S)]

    def leg_a(self):
        for s, (T, fit, conv, it, ns, nt) in zip(self.S, self.solo_out):
            rc = self.lib.liliom_loop_align(s.c._h, ptr(s.src_ids, C.c_int), ptr(s.src_poses, C.c_double), 1, ptr(s.tgt_ids, C.c_int),
                                            ptr(s.tgt_poses, C.c_double), LC_HIST, LC_LEAF, 30.0, 100, 1e-6, 1e-6, T, fit, conv, it, ns, nt)
            assert rc == 0, rc

    def leg_b(self):
        B = len(self.S)
        rc = self.lib.liliom_loop_align_batch(self.handles, B, self.si, self.sp, ptr(self.ks, C.c_int), self.ti, self.tp, ptr(self.kt, C.c_int),
                                              self.prm, self.out, ptr(self.status, C.c_int))
        assert rc == 0 and not self.status.any(), (rc, self.status)
        for s, r in zip(self.S, self.out):
            C.memmove(C.addressof(s.res["b"]), C.addressof(r), C.sizeof(r))

    def outputs(self, leg):
        out = b""
        for s in self.S:
            out += bytes(s.res[leg])
            C.memset(C.addressof(s.res[leg]), 0, C.sizeof(s.res[leg]))
        return out

    def prepare(self, leg):
        pass


HO_TRANS = (0.31, -0.12, 0.05)           # publishCloudLast's relative translation; the reference passes the identity rotation
HO_FLEETS = {"horizon": lambda i: 0, "hdl64": lambda i: 1, "mixed": lambda i: i % 2}


def handoff_sweep(args):
    from liliom_b200 import synth
    variant, seed = args
    T = synth.default_true_pose()
    if variant == 0:
        return synth.make_horizon_sweep(T, seed=seed)
    return synth.make_hdl64_sweep(T, seed=seed)


class HandoffSession:
    def __init__(self, variant, sweep):
        import liliom_b200 as L
        self.variant, (self.pts, q) = variant, sweep
        self.q = np.asarray(q, np.float64)
        self.bp = L.backend_default_params(variant)
        self.odo = L.Context(variant=variant)
        self.bk = {leg: L.Context(variant=variant) for leg in "ab"}
        self.odo.upload_scan(self.pts)           # the resident sweep; every tick re-extracts it
        self.res = {leg: np.zeros(5, np.int32) for leg in "ab"}     # kf_id, 3 counts, status of the leg's last tick

    def grow(self, keyframes):
        """both legs' arenas grown to `keyframes` hand-offs, then emptied: no timed call reallocates"""
        for bk in self.bk.values():
            for _ in range(keyframes):
                self.odo.extract_resident(self.q)
                self.odo.undistort_resident(HO_TRANS)
                bk.kf_add_resident(self.bp, self.odo)
            bk.kf_clear()

    def close(self):
        for c in (self.odo, *self.bk.values()):
            c.close()


class HandoffFleet:
    """B sessions and the C arguments of both legs, built once."""

    def __init__(self, S):
        import liliom_b200 as L
        self.S, self.lib, B = S, L._binding.lib(), len(S)
        for s in S:
            for bk in s.bk.values():
                bk.kf_clear()
        self.odos = (C.c_void_p * B)(*[s.odo._h for s in S])
        self.bks = {leg: (C.c_void_p * B)(*[s.bk[leg]._h for s in S]) for leg in "ab"}
        self.trans = np.tile(np.array(HO_TRANS), B)
        self.quat = np.tile(np.array([1.0, 0, 0, 0]), B)
        self.bps = (L.BackendParams * B)(*[s.bp for s in S])
        self.out = np.zeros((5, B), np.int32)     # kf_id, n_edge_ds, n_surf_ds, n_full_stored, status
        self.t, self.q = ptr(np.array(HO_TRANS), C.c_double), ptr(np.array([1.0, 0, 0, 0]), C.c_double)
        self.solo_out = [[ptr(s.res["a"][k:], C.c_int) for k in range(4)] for s in S]

    def prepare(self, leg):
        for s in self.S:
            s.odo.extract_resident(s.q)

    def leg_a(self):
        for s, (kid, ne, ns, nf) in zip(self.S, self.solo_out):
            rc = self.lib.liliom_undistort_resident(s.odo._h, self.t, self.q)
            rc = rc or self.lib.liliom_kf_add_resident(s.bk["a"]._h, C.byref(s.bp), s.odo._h, kid, ne, ns, nf)
            assert rc == 0, rc

    def leg_b(self):
        B = len(self.S)
        st = self.out[4]
        rc = self.lib.liliom_undistort_resident_batch(self.odos, B, ptr(self.trans, C.c_double), ptr(self.quat, C.c_double), ptr(st, C.c_int))
        assert rc == 0 and not st.any(), (rc, st)
        o = [np.ascontiguousarray(self.out[k]) for k in range(4)]
        rc = self.lib.liliom_kf_add_resident_batch(self.bks["b"], B, self.bps, self.odos, *[ptr(x, C.c_int) for x in o], ptr(st, C.c_int))
        assert rc == 0 and not st.any(), (rc, st)
        for i, s in enumerate(self.S):
            s.res["b"][:4] = [x[i] for x in o]

    def outputs(self, leg):
        out = b"".join(s.res[leg].tobytes() for s in self.S)
        for s in self.S:
            s.res[leg][:] = 0
        return out

    def stores(self, leg):
        """every session's last stored keyframe: its surf and full clouds as stored, and the store's size"""
        import liliom_b200 as L
        out = b""
        for s in self.S:
            bk = s.bk[leg]
            n = bk.kf_count()
            out += np.int32(n).tobytes()
            for kind in (L.KF_SURF, L.KF_FULL):
                out += bk.global_map(kind, [n - 1], [[1.0, 0, 0, 0, 0, 0, 0]], 1e-4).tobytes()
        return out


LM_FLEETS = {"horizon": lambda i: 0, "rot": lambda i: 1, "mixed": lambda i: i % 2}


def lm_stream(args):
    from liliom_b200 import synth
    variant, seed = args
    return synth.make_keyframe_sequence(NKF, stride=48 if variant == 0 else 32, seed=seed)


class LocalMapSession:
    """one session's store on a context per leg, the 40-keyframe list, and the window step's arguments (as Session's)"""

    def __init__(self, variant, seq):
        import liliom_b200 as L
        self.variant, self.bp = variant, L.backend_default_params(variant)
        self.c = {leg: L.Context(variant=variant) for leg in "ab"}
        for c in self.c.values():
            for e, s, _ in seq:
                c.kf_add(self.bp, e, s, download=False)
        self.base = [p for _, _, p in seq]
        self.ids = np.arange(NKF, dtype=np.int32)
        self.poses = {leg: np.zeros((NKF, 7)) for leg in "ab"}       # the tick's list poses, written in place by prepare
        self.tick = {leg: 0 for leg in "ab"}
        self.counts = {leg: np.zeros(2, np.int32) for leg in "ab"}
        self.win_ids = np.arange(NKF - WIN, NKF, dtype=np.int32)
        self.poses_l = np.array([nudge(seq[i][2], 1) for i in self.win_ids])
        self.bodies = [np.array([nudge(p, 2 + j) for p in self.poses_l]) for j in range(EVALS)]
        self.res = {leg: (np.zeros(WIN, np.int32), np.zeros(WIN, np.int32), [np.zeros((WIN, 2, 29)) for _ in range(EVALS)]) for leg in "ab"}

    def close(self):
        for c in self.c.values():
            c.close()


class LocalMapFleet:
    """B sessions and the C arguments of both legs, built once; step=True adds the window search and the 16 block evaluations"""

    def __init__(self, S, step):
        import liliom_b200 as L
        self.S, self.lib, self.step, B = S, L._binding.lib(), step, len(S)
        P, D = C.POINTER(C.c_int), C.POINTER(C.c_double)
        self.handles = {leg: (C.c_void_p * B)(*[s.c[leg]._h for s in S]) for leg in "ab"}
        self.bps = (L.BackendParams * B)(*[s.bp for s in S])
        self.ids = (P * B)(*[ptr(s.ids, C.c_int) for s in S])
        self.poses = (D * B)(*[ptr(s.poses["b"], C.c_double) for s in S])
        self.k = np.full(B, NKF, np.int32)
        self.ne_map, self.ns_map = np.zeros(B, np.int32), np.zeros(B, np.int32)
        self.win_ids = (P * B)(*[ptr(s.win_ids, C.c_int) for s in S])
        self.win_poses = (D * B)(*[ptr(s.poses_l, C.c_double) for s in S])
        self.kw = np.full(B, WIN, np.int32)
        self.ne = (P * B)(*[ptr(s.res["b"][0], C.c_int) for s in S])
        self.ns = (P * B)(*[ptr(s.res["b"][1], C.c_int) for s in S])
        self.bodies = [(D * B)(*[ptr(s.bodies[j], C.c_double) for s in S]) for j in range(EVALS)]
        self.outs = [(D * B)(*[ptr(s.res["b"][2][j], C.c_double) for s in S]) for j in range(EVALS)]
        self.status = np.zeros(B, np.int32)

    def prepare(self, leg):
        for s in self.S:
            t = s.tick[leg]
            s.poses[leg][:] = [nudge(p, t % 5) for p in s.base]
            s.tick[leg] = t + 1

    def leg_a(self):
        for s in self.S:
            h, cnt = s.c["a"]._h, s.counts["a"]
            rc = self.lib.liliom_bmap_build(h, C.byref(s.bp), ptr(s.ids, C.c_int), ptr(s.poses["a"], C.c_double), NKF, ptr(cnt, C.c_int),
                                            ptr(cnt[1:], C.c_int))
            assert rc == 0, rc
            if not self.step:
                continue
            ne, ns, out = s.res["a"]
            rc = self.lib.liliom_backend_window_correspond(h, C.byref(s.bp), ptr(s.win_ids, C.c_int), ptr(s.poses_l, C.c_double), WIN,
                                                           ptr(ne, C.c_int), ptr(ns, C.c_int))
            assert rc == 0, rc
            for j in range(EVALS):
                rc = self.lib.liliom_backend_window_blocks(h, ptr(s.bodies[j], C.c_double), WIN, ptr(out[j], C.c_double))
                assert rc == 0, rc

    def leg_b(self):
        B, st, h = len(self.S), ptr(self.status, C.c_int), self.handles["b"]
        rc = self.lib.liliom_bmap_build_batch(h, B, self.bps, self.ids, self.poses, ptr(self.k, C.c_int), ptr(self.ne_map, C.c_int),
                                              ptr(self.ns_map, C.c_int), st)
        assert rc == 0 and not self.status.any(), (rc, self.status)
        for i, s in enumerate(self.S):
            s.counts["b"][:] = (self.ne_map[i], self.ns_map[i])
        if not self.step:
            return
        rc = self.lib.liliom_backend_window_correspond_batch(h, B, self.bps, self.win_ids, self.win_poses, ptr(self.kw, C.c_int), self.ne,
                                                             self.ns, st)
        assert rc == 0 and not self.status.any(), (rc, self.status)
        for j in range(EVALS):
            rc = self.lib.liliom_backend_window_blocks_batch(h, B, self.bodies[j], ptr(self.kw, C.c_int), self.outs[j], st)
            assert rc == 0 and not self.status.any(), (rc, self.status)

    def outputs(self, leg):
        """leg's counts (and window results) of every session as bytes; cleared for the next step"""
        out = b""
        for s in self.S:
            ne, ns, blocks = s.res[leg]
            out += s.counts[leg].tobytes() + ne.tobytes() + ns.tobytes() + b"".join(o.tobytes() for o in blocks)
            for a in [s.counts[leg], ne, ns] + blocks:
                a.fill(0)
        return out

    def layers(self, leg):
        return b"".join(s.c[leg].bmap_download(layer).tobytes() for s in self.S for layer in (0, 1))


def timed(f, leg, steps):
    """median ms of `steps` window steps of leg "a" or "b", and the outputs of the last (every call returns with its sessions'
    work complete)"""
    import torch
    run = f.leg_a if leg == "a" else f.leg_b
    lat = []
    for _ in range(steps):
        f.outputs(leg)
        f.prepare(leg)
        torch.cuda.synchronize()
        t = time.perf_counter()
        run()
        lat.append((time.perf_counter() - t) * 1e3)
    return float(np.median(lat)), f.outputs(leg)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, nargs="*", default=[1, 2, 4, 8, 16, 32])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop", action="store_true", help="the fleet loop-closure tick instead of the window step")
    ap.add_argument("--handoff", action="store_true", help="the fleet keyframe hand-off tick instead of the window step")
    ap.add_argument("--localmap", action="store_true", help="the fleet backend local map (and keyframe step) instead of the window step")
    args = ap.parse_args()
    if args.loop:
        return main_loop(args)
    if args.handoff:
        return main_handoff(args)
    if args.localmap:
        return main_localmap(args)
    Bmax = max(args.sessions)
    with ProcessPoolExecutor(max_workers=min(Bmax, os.cpu_count() or 1)) as ex:     # the streams, before CUDA starts here
        seqs = list(ex.map(stream, [100 + s for s in range(Bmax)]))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("backend_batch_bench.py measures on a CUDA device; none is visible")
    print(json.dumps(dict(card(), keyframes=NKF, window=WIN, evals=EVALS, steps=args.steps, rounds=args.rounds,
                          figures="[median of rounds, min round, max round], ms per fleet window step")), flush=True)
    sessions = [Session(seq) for seq in seqs]
    for B in args.sessions:
        S = sessions[:B]
        f = Fleet(S)
        for leg in "ab":
            timed(f, leg, args.warmup)
        ra, rb, same = [], [], True
        for _ in range(args.rounds):
            ta, oa = timed(f, "a", args.steps)
            tb, ob = timed(f, "b", args.steps)
            ra.append(ta); rb.append(tb)
            same = same and oa == ob
        row = dict(sessions=B, edge_map=int(np.median([s.c.bmap_download(0).size for s in S])),
                   surf_map=int(np.median([s.c.bmap_download(1).size for s in S])),
                   a_solo_ms=spread(ra), b_batch_ms=spread(rb), a_waits=B * (1 + EVALS), b_waits=1 + EVALS,
                   speedup=round(float(np.median(ra) / np.median(rb)), 3), identical=bool(same))
        print(json.dumps(row), flush=True)
    for s in sessions:
        s.c.close()


def main_loop(args):
    Bmax = max(args.sessions)
    with ProcessPoolExecutor(max_workers=min(Bmax, os.cpu_count() or 1)) as ex:
        seqs = list(ex.map(loop_stream, [200 + s for s in range(Bmax)]))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("backend_batch_bench.py measures on a CUDA device; none is visible")
    print(json.dumps(dict(card(), leg="loop", history=LC_HIST, leaf=LC_LEAF, steps=args.steps, rounds=args.rounds,
                          figures="[median of rounds, min round, max round], ms per fleet loop-closure tick")), flush=True)
    sessions = [LoopSession(seq) for seq in seqs]
    for B in args.sessions:
        S = sessions[:B]
        f = LoopFleet(S)
        for leg in "ab":
            timed(f, leg, args.warmup)
        ra, rb, same = [], [], True
        for _ in range(args.rounds):
            ta, oa = timed(f, "a", args.steps)
            tb, ob = timed(f, "b", args.steps)
            ra.append(ta); rb.append(tb)
            same = same and oa == ob
        f.leg_a()
        rs = [s.res["a"] for s in S]
        row = dict(sessions=B, n_src=[min(r.n_src for r in rs), max(r.n_src for r in rs)], n_tgt=[min(r.n_tgt for r in rs), max(r.n_tgt for r in rs)],
                   iters=[min(r.iters for r in rs), max(r.iters for r in rs)],
                   a_solo_ms=spread(ra), b_batch_ms=spread(rb), a_waits=4 * B, b_waits=3,
                   speedup=round(float(np.median(ra) / np.median(rb)), 3), identical=bool(same))
        f.outputs("a")
        print(json.dumps(row), flush=True)
    for s in sessions:
        s.c.close()


def main_handoff(args):
    Bmax = max(args.sessions)
    jobs = [(v, 300 + 2 * s + v) for s in range(Bmax) for v in (0, 1)]
    with ProcessPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1)) as ex:
        sw = dict(zip(jobs, ex.map(handoff_sweep, jobs)))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("backend_batch_bench.py measures on a CUDA device; none is visible")
    print(json.dumps(dict(card(), leg="handoff", steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                          figures="[median of rounds, min round, max round], ms per fleet hand-off tick")), flush=True)
    ticks = args.warmup + args.rounds * args.steps + 1
    for fleet, variant_of in HO_FLEETS.items():
        sessions = [HandoffSession(variant_of(s), sw[variant_of(s), 300 + 2 * s + variant_of(s)]) for s in range(Bmax)]
        for s in sessions:
            s.grow(ticks)
        for B in args.sessions:
            S = sessions[:B]
            f = HandoffFleet(S)
            for leg in "ab":
                timed(f, leg, args.warmup)
            ra, rb, same = [], [], True
            for _ in range(args.rounds):
                ta, oa = timed(f, "a", args.steps)
                tb, ob = timed(f, "b", args.steps)
                ra.append(ta); rb.append(tb)
                same = same and oa == ob
            same = same and f.stores("a") == f.stores("b")
            n_hz = sum(1 for s in S if s.variant == 0)
            # the waits follow from the calls' structure (include/liliom.h); the run does not count them
            row = dict(fleet=fleet, sessions=B, a_solo_ms=spread(ra), b_batch_ms=spread(rb),
                       waits_by_design=[5 * B, 1 + (3 if n_hz else 2)],
                       speedup=round(float(np.median(ra) / np.median(rb)), 3), identical=bool(same))
            print(json.dumps(row), flush=True)
        for s in sessions:
            s.close()


def main_localmap(args):
    Bmax = max(args.sessions)
    jobs = [(v, 400 + 2 * s + v) for s in range(Bmax) for v in (0, 1)]
    with ProcessPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1)) as ex:
        seqs = dict(zip(jobs, ex.map(lm_stream, jobs)))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("backend_batch_bench.py measures on a CUDA device; none is visible")
    print(json.dumps(dict(card(), leg="localmap", keyframes=NKF, window=WIN, evals=EVALS, steps=args.steps, warmup=args.warmup,
                          rounds=args.rounds, figures="[median of rounds, min round, max round], ms per fleet tick")), flush=True)
    for fleet, variant_of in LM_FLEETS.items():
        sessions = [LocalMapSession(variant_of(s), seqs[variant_of(s), 400 + 2 * s + variant_of(s)]) for s in range(Bmax)]
        for B in args.sessions:
            S = sessions[:B]
            for step in (False, True):
                f = LocalMapFleet(S, step)
                for leg in "ab":
                    timed(f, leg, args.warmup)
                ra, rb, same = [], [], True
                for _ in range(args.rounds):
                    ta, oa = timed(f, "a", args.steps)
                    tb, ob = timed(f, "b", args.steps)
                    ra.append(ta); rb.append(tb)
                    same = same and oa == ob
                same = same and f.layers("a") == f.layers("b")
                # the waits follow from the calls' structure (include/liliom.h); the run does not count them: a solo local map with
                # both layers non-empty waits five times, the batch three; a window search and a blocks call wait once each
                per = 1 + EVALS if step else 0
                row = dict(fleet=fleet, sessions=B, call="keyframe_step" if step else "local_map",
                           edge_map=int(np.median([s.c["a"].bmap_download(0).size for s in S])),
                           surf_map=int(np.median([s.c["a"].bmap_download(1).size for s in S])),
                           a_solo_ms=spread(ra), b_batch_ms=spread(rb), waits_by_design=[B * (5 + per), 3 + per],
                           speedup=round(float(np.median(ra) / np.median(rb)), 3), identical=bool(same))
                print(json.dumps(row), flush=True)
        for s in sessions:
            s.close()


if __name__ == "__main__":
    main()
