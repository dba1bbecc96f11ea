#!/usr/bin/env python
"""ROT-package ingest of the spinning LiDAR's PointCloud2 (SURVEY §8 f3): host decode + the 32-byte path against the device decode.

For each synthetic driver layout (synth.PC2_LAYOUTS, the seeded 130k-point HDL-64E sweep) one step is
  (i)  a NumPy decode of the message into a pinned PointXYZI array (standing in for pcl::fromROSMsg on the node's host; PCL is
       not used here, so this is not PCL's cost) + liliom_extract_rot on it, or
  (ii) liliom_extract_rot_pc2 on the message payload, from the message's own (pageable) buffer and from a pinned copy of it.
Every call is synchronous (the library drains its stream before it returns), so a host clock around each call is the step time.
Reports the median step time of each path (and of the NumPy decode and of liliom_extract_rot on the decoded pinned cloud alone),
the host-to-device bytes per sweep, and whether (i) and (ii) give the same bytes.
Ring-field leg (LILIOM_RING_FIELD, the scanID read from the message's `ring` field): liliom_extract_rot_pc2 from a pinned payload
on a 128-ring x 1024-column Ouster-like sweep (packed u16 ring and organised u8 ring, line_num 128) and on the 64-ring HDL sweep
(line_num 64), each at ds_rate 4 (the ROT default) and 1.
Time-field leg (LILIOM_TIME_FIELD, relTime from the message's per-point time field): liliom_extract_rot_pc2 from a pinned payload
on the 128 x 1024 sweep as velodyne22 (`time`), ouster48 (`t`) and hesai26 (`timestamp`), ring field, line_num 128, ds_rate 4,
with the azimuth rule and with the time field on the same message, alternated in rounds so that both see the same clock drift.
The card's name and power limit are printed with the numbers.
usage: pc2_ingest_bench.py [--steps K] [--warmup W] [--out FILE]"""
import argparse
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

F32 = 7


def pinned(nbytes):
    import torch
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True).numpy()


def host_decode(msg, out):
    """pcl::fromROSMsg(msg, PointXYZI) with NumPy: out (PT32, n points) gets x, y, z, intensity from the first FLOAT32 field of
    each name with count 0 or 1 (0 when none), w = 1, padding 0.  One strided copy per field, no Python loop over points."""
    n = msg.width * msg.height
    o = out[:n]
    o[...] = np.zeros(1, L.PT32)
    o["w"] = 1.0
    for name in ("x", "y", "z", "intensity"):
        hit = [f for f in msg.fields if f[0] == name and f[2] == F32 and f[3] in (0, 1)]
        if not hit or n == 0:
            continue
        src = np.ndarray((msg.height, msg.width), "<f4", buffer=msg.data, offset=hit[0][1], strides=(msg.row_step, msg.point_step))
        dst = o[name].reshape(msg.height, msg.width)
        dst[...] = src
    return o


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the numbers are still printed; the power limit is then reported as unknown
        q = f"unknown ({e})"
    return name, q


def median_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    a = ap.parse_args()
    name, power = card()
    print(f"card: {name}; power limit, max SM clock: {power}", flush=True)
    T = synth.default_true_pose()
    pts, q_imu, ring, step = synth.make_hdl64_sweep(T, grid=True)
    q_lb = np.array([1.0, 0.0, 0.0, 0.0])
    ctx = L.Context(variant=1)
    rows = []
    for layout in synth.PC2_LAYOUTS:
        msg = synth.encode_pc2(pts, ring, step, layout)
        n = msg.width * msg.height
        pin_msg = L.PC2(pinned(msg.data.size)[:msg.data.size], msg.height, msg.width, msg.point_step, msg.row_step, msg.fields)
        pin_msg.data[:] = msg.data
        cloud = pinned(n * 32)[:n * 32].view(L.PT32)
        outs = [[pinned(n * 32)[:n * 32].view(L.PT32) for _ in range(3)] for _ in range(2)]

        def path_host():
            host_decode(msg, cloud)
            return ctx.extract_rot(cloud, q_imu, q_lb, out=outs[0])

        def path_pc2(m):
            return ctx.extract_rot_pc2(m, q_imu, q_lb, out=outs[1])

        ref = [x.tobytes() for x in path_host()]
        same = [x.tobytes() for x in path_pc2(msg)] == ref and [x.tobytes() for x in path_pc2(pin_msg)] == ref
        t_dec = median_ms(lambda: host_decode(msg, cloud), a.steps, a.warmup)
        t_host = median_ms(path_host, a.steps, a.warmup)
        t_ext = median_ms(lambda: ctx.extract_rot(cloud, q_imu, q_lb, out=outs[0]), a.steps, a.warmup)    # (i) without its decode
        t_pg = median_ms(lambda: path_pc2(msg), a.steps, a.warmup)
        t_pn = median_ms(lambda: path_pc2(pin_msg), a.steps, a.warmup)
        row = dict(layout=layout, points=n, point_step=msg.point_step, h2d_bytes_host_path=n * 32, h2d_bytes_pc2=msg.height * msg.row_step,
                   numpy_decode_ms=t_dec[0], extract_rot_pinned_pt32_ms=t_ext[0], host_decode_plus_extract_rot_ms=t_host[0],
                   extract_rot_pc2_pageable_ms=t_pg[0], extract_rot_pc2_pinned_ms=t_pn[0], min_max_ms={"host": t_host[1:], "pc2_pageable": t_pg[1:], "pc2_pinned": t_pn[1:]},
                   outputs_identical=bool(same), steps=a.steps, warmup=a.warmup, card=name, power_limit_max_sm_clock=power)
        rows.append(row)
        print(json.dumps(row), flush=True)
    ctx.close()
    ring_rows = ring_leg(a, name, power)
    time_rows = time_leg(a, name, power)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows + ring_rows + time_rows:
                f.write(json.dumps(r) + "\n")
    print(f"\n{'layout':<14} {'B/pt in':>8} {'H2D host':>10} {'H2D pc2':>10} {'decode':>8} {'32B ext':>8} {'(i) host':>9} "
          f"{'(ii) pg':>8} {'(ii) pin':>9} same")
    for r in rows:
        print(f"{r['layout']:<14} {r['point_step']:>8} {r['h2d_bytes_host_path']:>10} {r['h2d_bytes_pc2']:>10} {r['numpy_decode_ms']:>8.3f} "
              f"{r['extract_rot_pinned_pt32_ms']:>8.3f} {r['host_decode_plus_extract_rot_ms']:>9.3f} {r['extract_rot_pc2_pageable_ms']:>8.3f} {r['extract_rot_pc2_pinned_ms']:>9.3f} "
              f"{r['outputs_identical']}")
    print(f"(ms, median of {a.steps} steps after {a.warmup} warm-up steps; {name}, power limit / max SM clock {power})")
    print(f"\n{'ring-field leg':<24} {'rings':>5} {'ds':>3} {'points':>7} {'H2D B':>9} {'pinned ms':>9} {'min':>7} {'max':>7} {'edge':>5} {'surf':>6}")
    for r in ring_rows:
        print(f"{r['sweep'] + ' ' + r['layout']:<24} {r['line_num']:>5} {r['ds_rate']:>3} {r['points']:>7} {r['h2d_bytes_pc2']:>9} "
              f"{r['extract_rot_pc2_pinned_ms']:>9.3f} {r['min_max_ms'][0]:>7.3f} {r['min_max_ms'][1]:>7.3f} {r['n_edge']:>5} {r['n_surf']:>6}")
    print(f"(ms, median of {a.steps} steps after {a.warmup} warm-up steps; {name}, power limit / max SM clock {power})")
    print(f"\n{'time-field leg':<24} {'field':>9} {'B/pt':>4} {'azimuth ms':>10} {'time ms':>8} {'delta us':>8} {'edge az/t':>10} {'surf az/t':>12}")
    for r in time_rows:
        print(f"{r['sweep'] + ' ' + r['layout']:<24} {r['time_field']:>9} {r['point_step']:>4} {r['azimuth_ms']:>10.3f} {r['time_field_ms']:>8.3f} "
              f"{(r['time_field_ms'] - r['azimuth_ms']) * 1e3:>8.1f} {str(r['n_edge']):>10} {str(r['n_surf']):>12}")
    print(f"(ms, median of {a.steps} steps after {a.warmup} warm-up steps; {name}, power limit / max SM clock {power})")
    if not all(r["outputs_identical"] for r in rows):
        sys.exit(1)


def ring_leg(a, name, power):
    """liliom_extract_rot_pc2 with the ring taken from the message (LILIOM_RING_FIELD), pinned payload: 128 x 1024 vs the HDL sweep."""
    T = synth.default_true_pose()
    p128, q128, r128, s128 = synth.make_spinning_sweep(T, synth.uniform_elevations(128), 1024)
    p64, q64, r64, s64 = synth.make_hdl64_sweep(T, grid=True)
    cases = [("128x1024", "velodyne22", synth.encode_pc2(p128, r128, s128, "velodyne22", steps=1024, lines=128), q128, 128),
             ("128x1024", "ouster48", synth.encode_pc2(p128, r128, s128, "ouster48", steps=1024, lines=128), q128, 128),
             ("hdl64", "velodyne22", synth.encode_pc2(p64, r64, s64, "velodyne22"), q64, 64)]
    rows = []
    q_lb = np.array([1.0, 0.0, 0.0, 0.0])
    for sweep, layout, msg, q, lines in cases:
        pin = L.PC2(pinned(msg.data.size)[:msg.data.size], msg.height, msg.width, msg.point_step, msg.row_step, msg.fields)
        pin.data[:] = msg.data
        n = msg.width * msg.height
        outs = [pinned(n * 32)[:n * 32].view(L.PT32) for _ in range(3)]
        for ds in (4, 1):
            prm = L.default_params(1)
            prm.line_num = lines; prm.ds_rate = ds
            ctx = L.Context(prm)
            ctx.set_ring_source(L.RING_FIELD)
            surf, edge, _ = ctx.extract_rot_pc2(pin, q, q_lb, out=outs)
            t = median_ms(lambda: ctx.extract_rot_pc2(pin, q, q_lb, out=outs), a.steps, a.warmup)
            row = dict(leg="ring_field", sweep=sweep, layout=layout, line_num=lines, ds_rate=ds, points=n, point_step=msg.point_step,
                       h2d_bytes_pc2=msg.height * msg.row_step, extract_rot_pc2_pinned_ms=t[0], min_max_ms=t[1:], n_edge=len(edge),
                       n_surf=len(surf), steps=a.steps, warmup=a.warmup, card=name, power_limit_max_sm_clock=power)
            rows.append(row)
            print(json.dumps(row), flush=True)
            ctx.close()
    return rows


def time_leg(a, name, power):
    """liliom_extract_rot_pc2 with relTime from the azimuth rule vs from the message's time field (LILIOM_TIME_FIELD), pinned
    payload, same message: the 128 x 1024 sweep as velodyne22, ouster48 and hesai26 (ring field, line_num 128, ds_rate 4)."""
    T = synth.default_true_pose()
    p128, q128, r128, s128 = synth.make_spinning_sweep(T, synth.uniform_elevations(128), 1024)
    q_lb = np.array([1.0, 0.0, 0.0, 0.0])
    rows = []
    for layout in ("velodyne22", "ouster48", "hesai26"):
        msg = synth.encode_pc2(p128, r128, s128, layout, steps=1024, lines=128)
        pin = L.PC2(pinned(msg.data.size)[:msg.data.size], msg.height, msg.width, msg.point_step, msg.row_step, msg.fields)
        pin.data[:] = msg.data
        n = msg.width * msg.height
        field = synth.PC2_TIME_FIELDS[layout]
        ctxs, outs, counts = [], [], []
        for timed in (False, True):
            prm = L.default_params(1)
            prm.line_num = 128; prm.ds_rate = 4
            ctx = L.Context(prm)
            ctx.set_ring_source(L.RING_FIELD)
            if timed:
                ctx.set_time_source(L.TIME_FIELD, field)
            out = [pinned(n * 32)[:n * 32].view(L.PT32) for _ in range(3)]
            surf, edge, _ = ctx.extract_rot_pc2(pin, q128, q_lb, out=out)
            ctxs.append(ctx); outs.append(out); counts.append((len(edge), len(surf)))
        # alternate the two modes in rounds of 10 calls so that clock drift lands on both
        ts = [[], []]
        for k in range(a.warmup + a.steps):
            for j in (0, 1):
                t0 = time.perf_counter()
                ctxs[j].extract_rot_pc2(pin, q128, q_lb, out=outs[j])
                if k >= a.warmup:
                    ts[j].append((time.perf_counter() - t0) * 1e3)
        row = dict(leg="time_field", sweep="128x1024", layout=layout, time_field=field, line_num=128, ds_rate=4, points=n,
                   point_step=msg.point_step, h2d_bytes_pc2=msg.height * msg.row_step, azimuth_ms=float(np.median(ts[0])),
                   time_field_ms=float(np.median(ts[1])), min_max_ms={"azimuth": [min(ts[0]), max(ts[0])], "time_field": [min(ts[1]), max(ts[1])]},
                   n_edge=[counts[0][0], counts[1][0]], n_surf=[counts[0][1], counts[1][1]], steps=a.steps, warmup=a.warmup, card=name,
                   power_limit_max_sm_clock=power)
        rows.append(row)
        print(json.dumps(row), flush=True)
        for ctx in ctxs:
            ctx.close()
    return rows


if __name__ == "__main__":
    main()
