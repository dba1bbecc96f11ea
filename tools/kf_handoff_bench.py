#!/usr/bin/env python
"""One keyframe hand-off from the odometry to the backend (LidarOdometry::publishCloudLast -> BackendFusion's keyframe store),
timed both ways on the same resident clouds:
  host chain   liliom_features_download, liliom_undistort on the edge, surf and full clouds, liliom_kf_add, liliom_kf_add_full
               (seven calls, every cloud across PCIe four times), from pageable and from pinned host buffers;
  resident     liliom_undistort_resident + liliom_kf_add_resident (two calls, no cloud leaves the device).
Workloads: the seeded Horizon sweep (synth.make_horizon_sweep, 48-byte points, backend variant 0: the full cloud stored as
received) and the seeded HDL-64E sweep (synth.make_hdl64_sweep, 32-byte points, variant 1: VoxelGrid(surf_leaf) of the full
cloud), the sizes a user of each package sees.  The odometry context re-extracts the resident sweep before every hand-off (not
timed), so every hand-off starts from the same clouds; each path stores into a backend context of its own, the paths alternate
keyframe by keyframe, and the backends are emptied (liliom_kf_clear, untimed) every CLEAR_EVERY keyframes after a warm-up that
grew their arenas to that size, so that no timed call reallocates.  Every call is
synchronous, so a host clock around a hand-off is its time (the ctypes overhead of each call included: it is part of what a
caller pays).  Reports per path the median and the 10th / 90th percentiles, the cloud bytes each path moves across PCIe (from
the counts), and the kernel launches and library sort / scan calls (liliom_get_counters) of one hand-off.  Checks in the same
run that the stores the host chain and the resident calls build are bit-identical at these sizes.  The card's name and power
limit are printed with the numbers.
usage: kf_handoff_bench.py [--keyframes K] [--warmup W] [--out FILE]"""
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
import liliom_b200 as L                      # noqa: E402
from liliom_b200 import synth                # noqa: E402

IDENT_Q = np.array([1.0, 0.0, 0.0, 0.0])
IDENT7 = np.array([1.0, 0, 0, 0, 0, 0, 0])
TRANS = np.array([0.31, -0.12, 0.05])        # the scan's relative translation publishCloudLast de-skews with
TINY_LEAF = 1e-4                             # PCL declines the filter at this leaf: liliom_global_map returns the stored cloud
PATHS = ("host_pageable", "host_pinned", "resident")
CLEAR_EVERY = 200                            # keyframes per store between (untimed) kf_clear calls: ~200 MB of full clouds

dp, vp = C.POINTER(C.c_double), C.c_void_p


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    return q.stdout.strip() or f"nvidia-smi failed: {q.stderr.strip()}"


def pinned(n, dtype):
    import torch
    return torch.empty(max(n, 1) * dtype.itemsize, dtype=torch.uint8, pin_memory=True).numpy().view(dtype)


def _p(a):
    return a.ctypes.data_as(vp)


def _d(a):
    return a.ctypes.data_as(dp)


class Workload:
    def __init__(self, name, variant, pts, q):
        self.name, self.variant, self.pts, self.q = name, variant, pts, np.asarray(q, np.float64)
        self.odo = L.Context(variant=variant)
        self.bp = L.backend_default_params(variant)
        self.odo.upload_scan(pts)                                 # the resident sweep; every hand-off re-extracts it
        self.stride = self.odo.stride
        n = len(pts)
        self.bufs = {"host_pageable": [np.empty(max(n, 1), self.odo.dtype) for _ in range(3)],
                     "host_pinned": [pinned(n, self.odo.dtype) for _ in range(3)]}

    def extract(self):
        self.odo.extract_resident(self.q)

    def host(self, bk, bufs):
        """the seven-call chain; returns (kf_id, n_edge, n_surf, n_full) of what it sent"""
        lib = L._binding.lib()
        S, E, F = bufs
        ns, ne, nf = C.c_int(), C.c_int(), C.c_int()
        rc = lib.liliom_features_download(self.odo._h, _p(S), len(S), C.byref(ns), _p(E), len(E), C.byref(ne), _p(F), len(F), C.byref(nf))
        for buf, n in ((E, ne.value), (S, ns.value), (F, nf.value)):
            rc = rc or lib.liliom_undistort(self.odo._h, _p(buf), n, _d(TRANS), _d(IDENT_Q))
        kid, a, b, m = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        rc = rc or lib.liliom_kf_add(bk._h, C.byref(self.bp), _p(E), ne.value, _p(S), ns.value, C.byref(kid), None, 0, C.byref(a), None, 0, C.byref(b))
        rc = rc or lib.liliom_kf_add_full(bk._h, C.byref(self.bp), kid.value, _p(F), nf.value, C.byref(m))
        if rc:
            raise L.LiliomError(rc, "host chain")
        return kid.value, ne.value, ns.value, nf.value

    def resident(self, bk):
        lib = L._binding.lib()
        rc = lib.liliom_undistort_resident(self.odo._h, _d(TRANS), _d(IDENT_Q))
        kid, a, b, m = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        rc = rc or lib.liliom_kf_add_resident(bk._h, C.byref(self.bp), self.odo._h, C.byref(kid), C.byref(a), C.byref(b), C.byref(m))
        if rc:
            raise L.LiliomError(rc, "resident")
        return kid.value

    def run(self, path, bk):
        return self.resident(bk) if path == "resident" else self.host(bk, self.bufs[path])


def launches(cs):
    k = [c.counters() for c in cs]
    return sum(x.launches for x in k), sum(x.lib_launches for x in k)


def measure(w, K, W):
    bks = {p: L.Context(variant=w.variant) for p in PATHS}
    for _ in range(max(W, CLEAR_EVERY)):                          # warm-up, and arenas grown for CLEAR_EVERY keyframes
        for p in PATHS:
            w.extract()
            w.run(p, bks[p])
    times = {p: [] for p in PATHS}
    counts = None
    for r in range(K):
        if r % CLEAR_EVERY == 0:
            for bk in bks.values():
                bk.kf_clear()                                     # the arenas keep their allocations
        for j in range(len(PATHS)):
            p = PATHS[(r + j) % len(PATHS)]                       # alternate, and rotate which path goes first
            w.extract()
            t0 = time.perf_counter()
            out = w.run(p, bks[p])
            times[p].append(time.perf_counter() - t0)
            if p == "host_pageable":
                counts = out[1:]
    calls = {}
    for p in PATHS:                                               # the launches of one hand-off, counted on both contexts
        w.extract()
        for c in (w.odo, bks[p]):
            c.counters(reset=True)
        w.run(p, bks[p])
        calls[p] = launches([w.odo, bks[p]])
    for bk in bks.values():
        bk.close()
    ne, ns, nf = counts
    cloud = (ne + ns + nf) * w.stride
    res = {"workload": w.name, "stride": w.stride, "variant": w.variant, "n_sweep": len(w.pts), "n_edge": ne, "n_surf": ns,
           "n_full": nf, "keyframes": K, "pcie_cloud_bytes": {"host_pageable": 4 * cloud, "host_pinned": 4 * cloud, "resident": 0}}
    for p in PATHS:
        t = np.asarray(times[p]) * 1e3
        res[p] = {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)), "p90_ms": float(np.percentile(t, 90)),
                  "window_s": float(t.sum() / 1e3), "launches": calls[p][0], "lib_calls": calls[p][1]}
    return res


def store_parity(w, n_kf=8):
    """the host chain (pageable) into one backend, the resident calls into another, n_kf keyframes: identical stores?"""
    a, b = L.Context(variant=w.variant), L.Context(variant=w.variant)
    ok = True
    for _ in range(n_kf):
        w.extract()
        ra = w.host(a, w.bufs["host_pageable"])
        w.extract()
        kb = w.resident(b)
        ok &= ra[0] == kb
    ok &= a.kf_count() == b.kf_count() == n_kf
    for i in range(n_kf):
        for kind in (L.KF_SURF, L.KF_FULL):
            ok &= a.global_map(kind, [i], [IDENT7], TINY_LEAF).tobytes() == b.global_map(kind, [i], [IDENT7], TINY_LEAF).tobytes()
    ids = list(range(n_kf))
    poses = [IDENT7] * n_kf
    ok &= a.kf_cloud(ids, poses, 0.4).tobytes() == b.kf_cloud(ids, poses, 0.4).tobytes()
    a.close(); b.close()
    return bool(ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("kf_handoff_bench: no CUDA device (the measurement needs the GPU; there is no CPU path)")
    smi = card()
    T = synth.default_true_pose()
    hz, q_hz = synth.make_horizon_sweep(T)
    hdl, q_hdl = synth.make_hdl64_sweep(T)
    results = []
    for w in (Workload("horizon", 0, hz, q_hz), Workload("hdl64", 1, hdl, q_hdl)):
        r = measure(w, args.keyframes, args.warmup)
        r["stores_bit_identical"] = store_parity(w)
        w.odo.close()
        results.append(r)
        print(f"{r['workload']}: {r['n_sweep']} pts x {r['stride']} B, keyframe edge {r['n_edge']} surf {r['n_surf']} full {r['n_full']}; "
              f"stores bit-identical: {r['stores_bit_identical']}")
        for p in PATHS:
            x = r[p]
            print(f"  {p:14s} median {x['median_ms']:.3f} ms (p10 {x['p10_ms']:.3f}, p90 {x['p90_ms']:.3f}) over {r['keyframes']} keyframes "
                  f"({x['window_s']:.2f} s); PCIe cloud bytes {r['pcie_cloud_bytes'][p]}; launches {x['launches']} + {x['lib_calls']} sort/scan")
    print(f"card: {smi}")
    out = {"card": smi, "results": results}
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    if not all(r["stores_bit_identical"] for r in results):
        sys.exit("kf_handoff_bench: the two stores differ")


if __name__ == "__main__":
    main()
