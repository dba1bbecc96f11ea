"""Site map and cross-session loop closure over S stores (S = 2, 4, 8 by default) of K keyframes each: (a) the multi-store calls
(liliom_global_map_multi, liliom_loop_align_multi) against (b) the host route they replace: every store's transformed clouds
downloaded (liliom_global_map / liliom_kf_cloud at a declined leaf), joined on the host, uploaded again through liliom_voxelgrid,
and the loop's ICP run by liliom_icp_align.  The two are run alternately, each timed with a host clock around a call that ends in a
device synchronise, and must return identical bytes.  Prints one JSON line per S (median and spread over --reps) with the GPU's
name and power limit; --out also writes them to a file.

--fleet B... runs the fleet leg instead: B sessions (each a Horizon backend with a store of its own) share one prior store of --kf
keyframes.  Every session lists its own keyframes and a stretch of the prior map.  Timed, alternately, per B:
  (a) liliom_loop_align_batch_multi against B liliom_loop_align_multi calls;
  (b) liliom_bmap_build_batch_multi against B liliom_bmap_build_multi calls;
  (c) one liliom_bmap_build_multi against liliom_bmap_build on a merged store holding the same clouds (what reading across
      arenas costs).
Each pair must return identical bytes (loop results; counts and both layers).

    python tools/multi_store_bench.py [--stores 2 4 8] [--kf 300] [--leaf 0.4] [--reps 5] [--out multi_store.jsonl]
    python tools/multi_store_bench.py --fleet 1 2 4 8 16 32 [--kf 300] [--reps 7]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TINY_LEAF = 1e-4          # PCL declines the filter: the call returns the transformed concatenation


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:          # noqa: BLE001
        return f"unknown ({e})"


def build_stores(L, synth, S, K, bp):
    sweeps = synth.make_keyframe_sequence(12, stride=48, seed=3, full=True)
    T0 = synth.default_true_pose()
    stores, poses, n_in = [], {}, 0
    for s in range(S):
        c = L.Context(variant=0)
        for i in range(K):
            e, sf, _, f = sweeps[(7 * s + i) % len(sweeps)]
            kid, _, _ = c.kf_add(bp, e, sf, download=False)
            n_in += c.kf_add_full(bp, kid, f)
            q = synth.qmul(synth.q_from_axis_angle([0, 0, 1], np.deg2rad(1.0 * i + 90.0 * s)), T0[:4])
            poses[(s, i)] = np.concatenate([q, T0[4:] + np.array([1.5 * i, 40.0 * s, 0.0])])
        stores.append(c)
    return stores, poses, n_in


def timed(fn):
    t0 = time.perf_counter()
    out = fn()                      # every call below returns host bytes: it has synchronised the device
    return time.perf_counter() - t0, out


def stats(line, t):
    for k, v in t.items():
        line[f"{k}_ms_median"] = round(1e3 * float(np.median(v)), 3)
        line[f"{k}_ms_min"] = round(1e3 * float(np.min(v)), 3)
        line[f"{k}_ms_max"] = round(1e3 * float(np.max(v)), 3)
    return line


def fleet(L, synth, a, gpu):
    """the fleet leg: one JSON line per B"""
    bp = L.backend_default_params(0)
    seq = synth.make_keyframe_sequence(24, stride=48, seed=5)
    prior = L.Context(variant=0)
    prior_poses = []
    for i in range(a.kf):
        e, sf, p = seq[i % len(seq)]
        prior.kf_add(bp, e, sf, download=False)
        prior_poses.append(np.concatenate([p[:4], p[4:] + np.array([0.0, 30.0 * (i // len(seq)), 0.0])]))
    lines = []
    for B in a.fleet:
        sess, own = [], []
        for i in range(B):
            c = L.Context(variant=0)
            poses = []
            for j in range(6):
                e, sf, p = seq[(3 * i + j) % len(seq)]
                c.kf_add(bp, e, sf, download=False)
                poses.append(p)
            sess.append(c)
            own.append(poses)
        # session i: its own 6 keyframes and 24 prior keyframes around its place in the prior map; the loop: its latest keyframe
        # against 12 prior keyframes
        lists, loops = [], []
        for i in range(B):
            first = (37 * i) % (a.kf - 24)
            st = [sess[i]] * 6 + [prior] * 24
            ids = list(range(6)) + list(range(first, first + 24))
            ps = own[i] + prior_poses[first:first + 24]
            lists.append((st, ids, ps))
            loops.append(([sess[i]], [5], [own[i][5]], [prior] * 12, list(range(first + 6, first + 18)), prior_poses[first + 6:first + 18]))
        prm = dict(leaf=a.leaf, max_corr_dist=2.0, max_iter=50)

        def layers():
            return [c.bmap_download(l).tobytes() for c in sess for l in (0, 1)]

        def loop_batch():
            r, st = L.loop_align_batch_multi(sess, *[[x[k] for x in loops] for k in range(6)], [prm] * B)
            assert (st == 0).all()
            return [(x[0].tobytes(),) + tuple(x[1:]) for x in r]

        def loop_solo():
            return [(r[0].tobytes(),) + tuple(r[1:]) for r in (c.loop_align_multi(*x, **prm) for c, x in zip(sess, loops))]

        def bmap_batch():
            n, st = L.bmap_build_batch_multi(sess, [bp] * B, [x[0] for x in lists], [x[1] for x in lists], [x[2] for x in lists])
            assert (st == 0).all()
            return [tuple(r) for r in n.tolist()]

        def bmap_solo():
            return [tuple(c.bmap_build_multi(bp, *x)) for c, x in zip(sess, lists)]
        # (c): session 0's list on a merged store M (the prior store's adds, then session 0's)
        M = L.Context(variant=0)
        for i in range(a.kf):
            e, sf, _ = seq[i % len(seq)]
            M.kf_add(bp, e, sf, download=False)
        for j in range(6):
            e, sf, _ = seq[j % len(seq)]
            M.kf_add(bp, e, sf, download=False)
        m_ids = [a.kf + i for i in lists[0][1][:6]] + lists[0][1][6:]

        def merged():
            return M.bmap_build(bp, m_ids, lists[0][2])

        def across():
            return sess[0].bmap_build_multi(bp, *lists[0])
        for f in (loop_batch, loop_solo, bmap_batch, bmap_solo, merged, across):      # warm-up
            f()
        t = {k: [] for k in ("loop_batch", "loop_solo", "bmap_batch", "bmap_solo", "bmap_merged", "bmap_multi")}
        same_loop = same_bmap = same_merged = True
        for rep in range(a.reps):
            order = (0, 1) if rep % 2 == 0 else (1, 0)
            out = {}
            for k in order:
                name, fn = (("loop_batch", loop_batch), ("loop_solo", loop_solo))[k]
                dt, out[name] = timed(fn)
                t[name].append(dt)
            same_loop &= out["loop_batch"] == out["loop_solo"]
            for k in order:
                name, fn = (("bmap_batch", bmap_batch), ("bmap_solo", bmap_solo))[k]
                dt, r = timed(fn)
                t[name].append(dt)
                out[name] = (r, layers())
            same_bmap &= out["bmap_batch"] == out["bmap_solo"]
            for k in order:
                name, fn = (("bmap_merged", merged), ("bmap_multi", across))[k]
                dt, r = timed(fn)
                t[name].append(dt)
                out[name] = (r, [c.bmap_download(l).tobytes() for c in ((M,) if name == "bmap_merged" else (sess[0],)) for l in (0, 1)])
            same_merged &= out["bmap_merged"] == out["bmap_multi"]
        line = stats(dict(leg="fleet", sessions=B, prior_kf=a.kf, listed_per_session=30, gpu=gpu, reps=a.reps, identical_loop=bool(same_loop),
                          identical_bmap=bool(same_bmap), identical_merged=bool(same_merged)), t)
        print(json.dumps(line), flush=True)
        lines.append(line)
        for c in sess + [M]:
            c.close()
    prior.close()
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fleet", type=int, nargs="+", default=None)
    ap.add_argument("--stores", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--kf", type=int, default=300)
    ap.add_argument("--leaf", type=float, default=0.4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import liliom_b200 as L
    from liliom_b200 import synth
    bp = L.backend_default_params(0)
    gpu = gpu_info()
    if a.fleet:
        lines = fleet(L, synth, a, gpu)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                for line in lines:
                    f.write(json.dumps(line) + "\n")
        sys.exit(0 if all(x["identical_loop"] and x["identical_bmap"] and x["identical_merged"] for x in lines) else 1)
    lines = []
    for S in a.stores:
        stores, poses, n_in = build_stores(L, synth, S, a.kf, bp)
        caller = L.Context(variant=0)
        helper = L.Context(variant=0)                    # the host route's filter and ICP context
        entries = [(s, i) for i in range(a.kf) for s in range(S)]
        ctxs, ids, ps = [stores[s] for s, _ in entries], [i for _, i in entries], [poses[e] for e in entries]
        src = [(S - 1, a.kf - 1)]
        tgt = [(s, i) for s in range(S - 1) for i in range(a.kf - 20, a.kf)]

        def map_multi():
            return caller.global_map_multi(L.KF_FULL, ctxs, ids, ps, a.leaf)

        def map_host():
            parts = [stores[s].global_map(L.KF_FULL, [i], [poses[(s, i)]], TINY_LEAF) for s, i in entries]
            return helper.voxelgrid(np.concatenate(parts), a.leaf)

        def loop_multi():
            r = caller.loop_align_multi([stores[s] for s, _ in src], [i for _, i in src], [poses[e] for e in src],
                                        [stores[s] for s, _ in tgt], [i for _, i in tgt], [poses[e] for e in tgt], a.leaf,
                                        max_corr_dist=2.0, max_iter=50)
            return r[:4]

        def loop_host():
            def cloud(lst):
                parts = [stores[s].kf_cloud([i], [poses[(s, i)]], TINY_LEAF) for s, i in lst]
                return helper.voxelgrid(np.concatenate(parts), a.leaf)
            T, fit, conv, it = helper.icp_align(cloud(src), cloud(tgt), max_corr_dist=2.0, max_iter=50)
            return T, fit, conv, it

        map_multi(); map_host(); loop_multi(); loop_host()          # warm-up: modules, buffers, library sort plans
        t = {k: [] for k in ("map_multi", "map_host", "loop_multi", "loop_host")}
        same_map = same_loop = True
        for _ in range(a.reps):
            dm, gm = timed(map_multi)
            dh, gh = timed(map_host)
            lm_t, lm = timed(loop_multi)
            lh_t, lh = timed(loop_host)
            t["map_multi"].append(dm); t["map_host"].append(dh); t["loop_multi"].append(lm_t); t["loop_host"].append(lh_t)
            same_map &= gm.tobytes() == gh.tobytes()
            same_loop &= lm[0].tobytes() == lh[0].tobytes() and tuple(lm[1:]) == tuple(lh[1:])
        line = dict(stores=S, kf_per_store=a.kf, leaf=a.leaf, map_points_in=n_in, map_out=len(gm), gpu=gpu, reps=a.reps,
                    identical_map=bool(same_map), identical_loop=bool(same_loop))
        for k, v in t.items():
            line[f"{k}_ms_median"] = round(1e3 * float(np.median(v)), 2)
            line[f"{k}_ms_min"] = round(1e3 * float(np.min(v)), 2)
            line[f"{k}_ms_max"] = round(1e3 * float(np.max(v)), 2)
        print(json.dumps(line), flush=True)
        lines.append(line)
        for c in stores + [caller, helper]:
            c.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")
    if not all(x["identical_map"] and x["identical_loop"] for x in lines):
        sys.exit(1)


if __name__ == "__main__":
    main()
