#!/usr/bin/env python
"""The backend's LiDAR step (SURVEY.md §8 f5) on one GPU: device-resident keyframe store + local map + window calls, against the
same step through the single-keyframe ABI and the 1-thread oracle composition.  Prints one JSON line.
usage: backend_bench.py [--steps K] [--warmup W] [--dump-outputs DIR] [--global-map [--gm-keyframes 300,2000]] [--loop]
--dump-outputs DIR writes the last timed step's layers and blocks of the device-resident leg as DIR/<name>.npy.
--global-map runs the global-map leg instead (publishCompleteMap over the stored full clouds, one JSON line).
--loop runs the loop-closure leg instead (liliom_loop_align against kf_cloud x2 + icp_align and the oracle, one JSON line)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def dump_outputs(d, arrays):
    os.makedirs(d, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(d, name + ".npy"), a)


BK_MAP_WIDTH = 40      # local_map_width (L/config/config_fr_iosb.yaml)
BK_WINDOW = 3          # slide_window_width
BK_EVALS = 16          # max_num_iter (15) LM evaluations + 1 for the marginalisation


def bench_backend(args):
    """One step of BackendFusion's LiDAR side (SURVEY.md §8 f5) per new keyframe, Horizon variant, on the
    seeded keyframe stream of synth.make_keyframe_sequence.  A step: store the new keyframe's received clouds (VoxelGrid on the
    device), build the local map over the latest 40 keyframes, download both layers (published every run), search the window's
    3 keyframes, evaluate the window's blocks 16 times (15 LM iterations + the marginalisation).
    Legs: (a) this path; (b) the same step through the single-keyframe ABI (host transform + concatenation in NumPy,
    liliom_voxelgrid x2, liliom_map_set_cloud on an edge and a surf context, then for each of the 16 evaluations and each window
    keyframe liliom_correspond_edge / _surf_refl + the block: one context holds one keyframe's correspondences at a time);
    (c) the 1-thread oracle composition of (b), on a bounded sample."""
    import torch
    import liliom_b200 as L
    from liliom_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("backend_bench.py needs a CUDA device (no CPU fallback)")
    name, plim = gpu_card()
    bp = L.backend_default_params(0)
    pool = synth.make_keyframe_sequence(BK_MAP_WIDTH + 8, stride=48)
    steps, warmup = args.steps, args.warmup
    q_lb, t_lb = np.array(bp.q_lb[:]), np.array(bp.t_lb[:])

    def body_of(p):         # inverse of :929-930, quaternion kept unit as Ceres' QuaternionParameterization keeps it
        q = synth.qmul(p[:4], q_lb)
        return np.concatenate([q / np.linalg.norm(q), p[4:] + synth.qrot(p[:4], t_lb)])

    def trial(p, it):       # LM trial poses: small deterministic steps
        dq = synth.q_from_axis_angle([1, -1, 2], np.deg2rad(0.01 * it))
        return np.concatenate([synth.qmul(p[:4], dq), p[4:] + 1e-3 * it])

    psz = 48
    # ---- (a) device-resident store and local map
    c = L.Context(variant=0)
    kf_pose = []
    for e, s, p in pool[:BK_MAP_WIDTH]:                        # a stream already BK_MAP_WIDTH keyframes long
        c.kf_add(bp, e, s, download=False); kf_pose.append(p)
    kf_sizes = []                                               # stored (edge, surf) points per keyframe, for leg (b)'s byte count

    def step_a(j):
        e, s, p = pool[j % len(pool)]
        kid, _, _ = c.kf_add(bp, e, s, download=False); kf_pose.append(p)
        ids = list(range(kid + 1 - BK_MAP_WIDTH, kid + 1))
        c.bmap_build(bp, ids, [kf_pose[i] for i in ids])
        em, sm = c.bmap_download(0), c.bmap_download(1)
        win = list(range(kid - BK_WINDOW, kid))                 # idx - 1
        pl = [kf_pose[i] for i in win]
        ne, ns = c.backend_window_correspond(bp, win, pl)
        blocks = [c.backend_window_blocks([trial(body_of(p), it) for p in pl]) for it in range(BK_EVALS)]
        h2d = (len(e) + len(s)) * psz
        d2h = (len(em) + len(sm)) * psz + BK_EVALS * BK_WINDOW * 2 * 29 * 8
        return (em, sm, blocks[-1]), h2d, d2h

    def timed(fn, n, w):
        for j in range(w):
            fn(j)
        ms, out = [], None
        for j in range(w, w + n):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(j)
            ms.append((time.perf_counter() - t0) * 1e3)
        return ms, out

    def stats(ms, out):
        return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)), "steps": len(ms),
                "h2d_bytes_per_step": int(out[1]), "d2h_bytes_per_step": int(out[2])}

    ms_a, out_a = timed(step_a, steps, warmup)
    # ---- (b) the single-keyframe ABI: the adapter keeps every keyframe cloud and builds the local map on the host
    cb, ce, cs = L.Context(variant=0), L.Context(variant=0), L.Context(variant=0)
    store = []                                                  # host copies of edge_frames / surf_frames (:1688-1695)
    pose_b = []
    for e, s, p in pool[:BK_MAP_WIDTH]:
        store.append((cb.voxelgrid(e, bp.edge_leaf), cb.voxelgrid(s, bp.surf_leaf))); pose_b.append(p)

    def host_transform(cloud, p):
        out = cloud.copy()
        xyz = np.stack([cloud["x"], cloud["y"], cloud["z"]], 1).astype(np.float64)
        w = synth._rotate_many(np.broadcast_to(p[:4], (len(xyz), 4)), xyz) + p[4:]
        n = synth._rotate_many(np.broadcast_to(p[:4], (len(xyz), 4)), np.stack([cloud["nx"], cloud["ny"], cloud["nz"]], 1).astype(np.float64))
        out["x"], out["y"], out["z"] = w[:, 0], w[:, 1], w[:, 2]
        out["nx"], out["ny"], out["nz"] = n[:, 0], n[:, 1], n[:, 2]
        return out

    def step_b(j):
        e, s, p = pool[j % len(pool)]
        eds, sds = cb.voxelgrid(e, bp.edge_leaf), cb.voxelgrid(s, bp.surf_leaf)
        store.append((eds, sds)); pose_b.append(p)
        kid = len(store) - 1
        h2d = (len(e) + len(s)) * psz; d2h = (len(eds) + len(sds)) * psz
        ids = range(kid + 1 - BK_MAP_WIDTH, kid + 1)
        E = np.concatenate([host_transform(store[i][0], pose_b[i]) for i in ids])
        S = np.concatenate([host_transform(store[i][1], pose_b[i]) for i in ids])
        em, sm = cb.voxelgrid(E, bp.edge_leaf), cb.voxelgrid(S, bp.surf_leaf)
        h2d += (len(E) + len(S)) * psz; d2h += (len(em) + len(sm)) * psz
        ce.map_set_cloud(em); cs.map_set_cloud(sm)
        h2d += (len(em) + len(sm)) * psz
        win = list(range(kid - BK_WINDOW, kid))
        pl = [pose_b[i] for i in win]
        blocks = np.zeros((BK_WINDOW, 2, 29))
        for it in range(BK_EVALS):
            for k, i in enumerate(win):
                fe, fs = store[i]
                v, _, _ = ce.correspond_edge(fe, pl[k], 0)
                blocks[k, 0] = ce.backend_edge_block(trial(body_of(pl[k]), it), float(np.float32(bp.lidar_const)), bp.cauchy_b)
                ve, _, _ = cs.correspond_surf_refl(fs, pl[k], bp.kd_max_radius, bp.surf_dist_thres, bp.w_gate, bp.lidar_const, bp.reflect_thres)
                blocks[k, 1] = cs.backend_surf_block(trial(body_of(pl[k]), it), q_lb, t_lb, bp.cauchy_b)
                h2d += (len(fe) + len(fs)) * psz
                d2h += len(fe) * 25 + len(fs) * 25 + 2 * 29 * 8
        return (em, sm, blocks), h2d, d2h

    ms_b, out_b = timed(step_b, steps, warmup)
    # ---- (c) 1-thread oracle composition of (b), bounded sample
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as O
    store_o = [(O.voxelgrid(e, bp.edge_leaf), O.voxelgrid(s, bp.surf_leaf)) for e, s, _ in pool[:BK_MAP_WIDTH]]
    pose_o = [p for _, _, p in pool[:BK_MAP_WIDTH]]

    def f4(a):
        return np.stack([a["x"], a["y"], a["z"], np.ones(len(a), np.float32)], 1)

    def step_c(j):
        e, s, p = pool[j % len(pool)]
        store_o.append((O.voxelgrid(e, bp.edge_leaf), O.voxelgrid(s, bp.surf_leaf))); pose_o.append(p)
        kid = len(store_o) - 1
        ids = range(kid + 1 - BK_MAP_WIDTH, kid + 1)
        em = O.voxelgrid(np.concatenate([O.transform_cloud(store_o[i][0], pose_o[i]) for i in ids]), bp.edge_leaf)
        sm = O.voxelgrid(np.concatenate([O.transform_cloud(store_o[i][1], pose_o[i]) for i in ids]), bp.surf_leaf)
        te, ts = O.KdTree(f4(em)), O.KdTree(f4(sm))
        win = list(range(kid - BK_WINDOW, kid))
        blocks = np.zeros((BK_WINDOW, 2, 29))
        corr = []
        for i in win:
            fe, fs = store_o[i]
            corr.append((O.correspond_edge(te, fe, pose_o[i], 0),
                         O.correspond_surf_backend(ts, fs, pose_o[i], bp.kd_max_radius, bp.surf_dist_thres, bp.w_gate, bp.lidar_const,
                                                   sm["curvature"], fs["curvature"], bp.reflect_thres)))
        for it in range(BK_EVALS):
            for k, i in enumerate(win):
                (v, pa, pb), (vs, pls, sc) = corr[k]
                b = trial(body_of(pose_o[i]), it)
                blocks[k, 0] = O.backend_edge_block(store_o[i][0], v, pa, pb, float(np.float32(bp.lidar_const)), b, bp.cauchy_b)
                blocks[k, 1] = O.backend_surf_block(store_o[i][1], vs, pls, sc, b, q_lb, t_lb, bp.cauchy_b)
        return (em, sm, blocks), 0, 0

    n_c = min(steps, 5)
    ms_c, out_c = timed(step_c, n_c, 0)
    n_edge, n_surf = len(out_a[0][0]), len(out_a[0][1])
    line = {
        "metric": "ms per BackendFusion LiDAR step (keyframe store + 40-keyframe local map + 3-keyframe window, 16 block evaluations)",
        "workload": "backend", "unit": "ms/step", "higher_is_better": False, "n_gpus": 1, "steps": steps, "warmup": warmup,
        "value": float(np.median(ms_a)), "gpu": name, "power_limit": plim, "data": "synthetic (synth.make_keyframe_sequence)",
        "config": {"variant": 0, "local_map_width": BK_MAP_WIDTH, "slide_window_width": BK_WINDOW, "block_evaluations": BK_EVALS,
                   "edge_layer_points": n_edge, "surf_layer_points": n_surf,
                   "keyframe_points_received": int(np.mean([len(e) + len(s) for e, s, _ in pool]))},
        "device_resident": stats(ms_a, out_a),
        "single_keyframe_abi": stats(ms_b, out_b),
        "oracle_1_thread": {**stats(ms_c, out_c), "h2d_bytes_per_step": None, "d2h_bytes_per_step": None,
                            "sample": f"{n_c} steps, 1 thread, correspondences searched once per window keyframe"},
        "timing": "host wall clock around each step (every library call ends in a stream synchronise)",
    }
    if args.dump_outputs:
        (em, sm, blk) = out_a[0]
        dump_outputs(args.dump_outputs, {"backend_edge_layer": em.view(np.float32).reshape(-1), "backend_surf_layer": sm.view(np.float32).reshape(-1),
                                         "backend_blocks": np.asarray(blk, np.float64)})
    print(json.dumps(line), flush=True)
    for x in (c, cb, ce, cs):
        x.close()


def gpu_card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        plim = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception as e:      # noqa: BLE001
        plim = "unknown (" + type(e).__name__ + ")"
    return name, plim


GM_LEAF = 0.3          # mapping_ds (L/src/BackendFusion.cpp:568)
GM_SWEEPS = 24         # distinct full sweeps, reused cyclically along the path


def bench_global_map(args):
    """publishCompleteMap (L/src/BackendFusion.cpp:2644-2685) over a whole trajectory: every keyframe's full cloud (~20k points,
    Horizon variant, stored as received) transformed by its pose, concatenated, VoxelGrid(mapping_ds = 0.3).  Per trajectory length:
    (a) liliom_global_map on the full clouds kept in the device store (one call, output downloaded);
    (b) what a host-side adapter does without it: host copies of the full clouds, transformed on one CPU thread (PCL's
        transformPointCloud: the oracle's transform_cloud), concatenated in NumPy, then liliom_voxelgrid (upload, filter, download);
    (c) the 1-thread oracle composition voxelgrid(concat(transform_cloud(...))).
    The path is synth.make_keyframe_sequence's (1.5 m and 2 deg of yaw per keyframe); GM_SWEEPS generated sweeps are reused."""
    import torch
    import ctypes as C
    import liliom_b200 as L
    from liliom_b200 import synth
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as O
    if not torch.cuda.is_available():
        raise SystemExit("backend_bench.py needs a CUDA device (no CPU fallback)")
    name, plim = gpu_card()
    sweeps = [kf[3] for kf in synth.make_keyframe_sequence(GM_SWEEPS, stride=48, full=True)]
    T0 = synth.default_true_pose()
    bp = L.backend_default_params(0)
    lengths = [int(x) for x in args.gm_keyframes.split(",")]
    steps = max(1, args.steps)
    legs = []
    for n_kf in lengths:
        poses = []
        for i in range(n_kf):
            q = synth.qmul(synth.q_from_axis_angle([0, 0, 1], np.deg2rad(2.0 * i)), T0[:4])
            poses.append(np.concatenate([q, T0[4:] + np.array([1.5 * i, 0.35 * np.sin(0.4 * i), 0.0])]))
        clouds = [sweeps[i % GM_SWEEPS] for i in range(n_kf)]
        n_in = int(sum(len(x) for x in clouds))
        c = L.Context(variant=0)
        empty = sweeps[0][:0]
        for x in clouds:
            kid, _, _ = c.kf_add(bp, empty, empty, download=False)
            c.kf_add_full(bp, kid, x)
        ids = np.arange(n_kf, dtype=np.int32)
        p7 = np.ascontiguousarray(np.stack(poses))
        out = np.zeros(n_in, L.PT48)
        m = C.c_int()

        def arm_a():
            c._check(L._binding.lib().liliom_global_map(c._h, L.KF_FULL, ids.ctypes.data_as(C.POINTER(C.c_int)),
                                                        p7.ctypes.data_as(C.POINTER(C.c_double)), n_kf, None, GM_LEAF,
                                                        out.ctypes.data_as(C.c_void_p), len(out), C.byref(m)))
            return out[:m.value]

        def arm_b():
            cat = np.concatenate([O.transform_cloud(x, p) for x, p in zip(clouds, poses)])
            return c.voxelgrid(cat, GM_LEAF)

        def arm_c():
            return O.voxelgrid(np.concatenate([O.transform_cloud(x, p) for x, p in zip(clouds, poses)]), GM_LEAF)

        def timed(fn, n):
            fn()                                                  # warm-up (allocations)
            ms, res = [], None
            for _ in range(n):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = fn()
                ms.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ms)), res

        ms_a, got_a = timed(arm_a, steps)
        ms_b, got_b = timed(arm_b, steps)
        t0 = time.perf_counter()
        got_c = arm_c()
        ms_c = (time.perf_counter() - t0) * 1e3
        same = got_a.tobytes() == got_b.tobytes() == got_c.tobytes()
        legs.append({"keyframes": n_kf, "points_in": n_in, "bytes_in": n_in * 48, "points_out": int(len(got_a)),
                     "pcl_declined": bool(len(got_a) == n_in), "outputs_bit_identical": bool(same),
                     "a_global_map_median_ms": ms_a, "b_host_transform_concat_voxelgrid_median_ms": ms_b,
                     "c_oracle_1_thread_ms": ms_c, "timed_runs_a_b": steps, "timed_runs_c": 1})
        del out
        c.close()
    line = {"metric": "ms per publishCompleteMap over the whole trajectory (full clouds, VoxelGrid 0.3 m)", "workload": "backend_global_map",
            "unit": "ms", "higher_is_better": False, "n_gpus": 1, "gpu": name, "power_limit": plim,
            "data": f"synthetic: {GM_SWEEPS} synth.make_keyframe_sequence full sweeps reused along the path", "legs": legs,
            "timing": "host wall clock around each call, output on the host; (b) includes the host transform and concatenation"}
    print(json.dumps(line), flush=True)


LC_HIST = 41           # his_key_frames_ds: 2 * lc_map_width (20) + 1 keyframes (L/src/BackendFusion.cpp:2502-2547)
LC_LEAF = 0.4          # the loop-closure clouds' VoxelGrid (:2494, :2545)


def bench_loop(args):
    """detectLoopClosure's clouds + performLoopClosure's ICP (L/src/BackendFusion.cpp:2473-2582) on a keyframe sequence whose end
    revisits its start (synth.make_keyframe_sequence(41, revisit=1)): source = the revisit keyframe, listed with a pose off by
    2 deg / 0.5 m (the drift a loop closure corrects), target = the 41 history keyframes; leaf 0.4, the reference's ICP settings
    (:2566-2570).  Three legs:
    (a) liliom_loop_align on the backend context (one call, both clouds stay on the device);
    (b) liliom_kf_cloud x2 to the host, then liliom_icp_align on a second context (the composition (a) replaces);
    (c) the 1-thread oracle composition voxelgrid(concat(transform_cloud(...))) x2 + the NumPy / kd-tree restatement of PCL's
        loop (tests/test_gpu_widen.py::_icp_numpy), a few calls."""
    import torch
    import liliom_b200 as L
    from liliom_b200 import synth
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as O
    from test_gpu_widen import _icp_numpy
    if not torch.cuda.is_available():
        raise SystemExit("backend_bench.py needs a CUDA device (no CPU fallback)")
    name, plim = gpu_card()
    seq = synth.make_keyframe_sequence(LC_HIST, stride=48, revisit=1)
    bp = L.backend_default_params(0)
    c = L.Context(variant=0)
    for e, s, _ in seq:
        c.kf_add(bp, e, s, download=False)
    c2 = L.Context(variant=0)
    poses = [p for _, _, p in seq]
    qd = synth.q_from_axis_angle([0.1, -0.1, 1.0], np.deg2rad(2.0))
    w, x, y, z = qd
    Rd = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                   [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                   [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    p_src = poses[LC_HIST]
    src_pose = np.concatenate([synth.qmul(qd, p_src[:4]), Rd @ p_src[4:] + np.array([0.4, -0.25, 0.15])])
    si, sp = [LC_HIST], [src_pose]
    ti, tp = list(range(LC_HIST)), poses[:LC_HIST]
    stride = 48

    def arm_a():
        return c.loop_align(si, sp, ti, tp, LC_LEAF)

    def arm_b():
        src = c.kf_cloud(si, sp, LC_LEAF)
        tgt = c.kf_cloud(ti, tp, LC_LEAF)
        T, fit, conv, it = c2.icp_align(src, tgt)
        return T, fit, conv, it, len(src), len(tgt)

    def oracle_cloud(ids, ps):
        return O.voxelgrid(np.concatenate([O.transform_cloud(np.concatenate([seq[i][0], seq[i][1]]), p) for i, p in zip(ids, ps)]), LC_LEAF)

    def arm_c():
        src, tgt = oracle_cloud(si, sp), oracle_cloud(ti, tp)
        f4 = lambda a: np.ascontiguousarray(np.stack([a["x"], a["y"], a["z"], np.ones(len(a), np.float32)], 1))
        T, fit, conv, it = _icp_numpy(O, f4(src), f4(tgt))
        return T, fit, conv, it, len(src), len(tgt)

    def timed(fn, n, warm):
        for _ in range(warm):
            fn()
        ms, res = [], None
        for _ in range(n):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fn()
            ms.append((time.perf_counter() - t0) * 1e3)
        return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)), "timed_runs": n}, res

    steps = max(1, args.steps)
    ta, ra = timed(arm_a, steps, max(1, args.warmup))
    tb, rb = timed(arm_b, steps, max(1, args.warmup))
    tc, rc = timed(arm_c, 3, 0)
    n_src, n_tgt = ra[4], ra[5]
    pts_src = sum(len(seq[i][0]) + len(seq[i][1]) for i in si)
    pts_tgt = sum(len(seq[i][0]) + len(seq[i][1]) for i in ti)
    legs = {
        "a_loop_align": dict(ta, iters=ra[3], converged=bool(ra[2]), fitness=ra[1], cloud_h2d_bytes=0, cloud_d2h_bytes=0),
        "b_kf_cloud_x2_icp_align_second_context": dict(tb, iters=rb[3], converged=bool(rb[2]), fitness=rb[1],
                                                        cloud_h2d_bytes=(n_src + n_tgt) * stride, cloud_d2h_bytes=(n_src + n_tgt) * stride),
        "c_oracle_composition_numpy_icp": dict(tc, iters=rc[3], converged=bool(rc[2]), fitness=rc[1]),
    }
    T_err = float(np.abs(rc[0] - ra[0]).max())
    line = {"metric": "ms per loop closure (both clouds from the keyframe store + ICP)", "workload": "backend_loop_closure", "unit": "ms",
            "higher_is_better": False, "n_gpus": 1, "gpu": name, "power_limit": plim,
            "data": f"synthetic: synth.make_keyframe_sequence({LC_HIST}, revisit=1), source 1 keyframe ({pts_src} points in, {n_src} after "
                    f"VoxelGrid {LC_LEAF}), target {len(ti)} keyframes ({pts_tgt} points in, {n_tgt} after)",
            "a_b_T16_bit_identical": bool(ra[0].tobytes() == rb[0].tobytes() and ra[1:] == rb[1:]),
            "a_vs_c_max_abs_T_diff": T_err, "legs": legs,
            "bytes": "cloud bytes crossing the host link per call (b: both filtered clouds down and up again); not counted: the "
                     "keyframe tables, the counts and the results, a few kB per call in both legs",
            "timing": "host wall clock around each call, results on the host"}
    print(json.dumps(line), flush=True)
    c.close(); c2.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", default="", metavar="DIR")
    ap.add_argument("--global-map", action="store_true", help="run the global-map leg instead of the LiDAR step")
    ap.add_argument("--gm-keyframes", default="300,2000", help="trajectory lengths of the global-map leg")
    ap.add_argument("--loop", action="store_true", help="run the loop-closure leg instead of the LiDAR step")
    args = ap.parse_args()
    if args.loop:
        bench_loop(args)
    elif args.global_map:
        bench_global_map(args)
    else:
        bench_backend(args)


if __name__ == "__main__":
    main()
