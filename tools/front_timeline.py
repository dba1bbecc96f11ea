#!/usr/bin/env python
"""Stage clocks of the front of the headline resident step (on the GPU).

Runs bench.py's default step (24k-pt Horizon sweep -> k_hz_coop -> k_vg_coop -> 10 GN passes against the 1 M-pt map,
L2 flushed between steps) with LILIOM_DEBUG_TIMING=1 in a child process, parses the lines the library prints to stderr
after every step and reports, per kernel, the median over the measured steps of
  - the stage cycles of block 0 ([k_hz_coop, ...], [k_vg_coop, ...]),
  - the [step timeline] spans (%globaltimer of block 0 of each kernel, ns),
together with the card's name, power limit and SM clock read in the same run.  LILIOM_LIB selects another build of the
library (e.g. the parent commit's), so two builds can be compared in one job.
usage: front_timeline.py [--steps N] [--warmup W] [--json FILE]"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ITERS = 10

CYCLE_LINE = re.compile(r"^\[(k_hz_coop|k_vg_coop), cycles, block 0\] (.*)$")
PAIR = re.compile(r"\s*([^,()|:]*?[A-Za-z][^,()|:]*?)\s+(-?\d+)\s*(?=[,()|]|$)")
TIMELINE = re.compile(r"^\[step timeline, ns from k_hz_coop start\] hz 0\.\.(-?\d+) \| gap (-?\d+) \| vg (-?\d+)\.\.(-?\d+) \| "
                      r"gap (-?\d+) \| gn (-?\d+)\.\.(-?\d+) \((-?\d+)\)")


def child(steps, warmup):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import liliom_b200 as L
    from liliom_b200 import synth
    m, _ = synth.make_map(1_000_000)
    T0 = synth.default_true_pose()
    sweeps = []
    for k in range(8):                                  # bench.py's sweeps
        T = np.array(T0); T[4] += 0.7 * k; T[5] += 0.15 * k
        pts, q = synth.make_horizon_sweep(T, seed=1 + k)
        sweeps.append((pts, q, synth.perturbed_pose(T)))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    c = L.Context(L.default_params(0))
    c.set_stream(stream.cuda_stream)
    c.map_set_points(m)
    ms = []
    with torch.cuda.stream(stream):
        for k in range(warmup + steps):
            pts, q, guess = sweeps[k % len(sweeps)]
            c.upload_scan(pts)
            flush.fill_(k & 0xff)
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            c.extract_resident(q)
            c.odometry_resident(guess, ITERS, mode=L.MODE_GN, want_stats=False)
            e1.record(stream); e1.synchronize()
            sys.stderr.flush()
            print(f"STEP {k} {e0.elapsed_time(e1) * 1e3:.1f}", file=sys.stderr, flush=True)
    c.close()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "", "lib": L.LIB_PATH}))


def parse(stderr, warmup):
    """Per-step records from the child's stderr; a step's lines precede its STEP marker."""
    cur, recs = {}, []
    for line in stderr.splitlines():
        if line.startswith("STEP "):
            _, k, us = line.split()
            cur["step_us (events)"] = float(us)
            if int(k) >= warmup:
                recs.append(cur)
            cur = {}
            continue
        mc = CYCLE_LINE.match(line)
        if mc:
            for lab, v in PAIR.findall(mc.group(2)):
                cur[f"{mc.group(1)} {lab.strip()}"] = int(v)
            continue
        mt = TIMELINE.match(line)
        if mt:
            hz, g1, vg0, vg1, g2, gn0, gn1, gn = (int(x) for x in mt.groups())
            cur.update({"span hz": hz, "gap hz->vg": g1, "span vg": vg1 - vg0, "gap vg->gn": g2, "span gn": gn, "step end": gn1})
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--json", default="", help="also write the medians to this file")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.steps, a.warmup)
        return
    if a.steps < 50:
        sys.exit("--steps must be >= 50")
    env = dict(os.environ, LILIOM_DEBUG_TIMING="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--steps", str(a.steps), "--warmup", str(a.warmup)],
                       env=env, capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(f"child failed ({r.returncode}):\n{r.stderr[-4000:]}")
    info = json.loads(r.stdout.strip().splitlines()[-1])
    recs = parse(r.stderr, a.warmup)
    keys = []
    for rec in recs:
        keys += [k for k in rec if k not in keys]
    med = {k: statistics.median(rec[k] for rec in recs if k in rec) for k in keys}
    print(f"{info['device']} | nvidia-smi name, power.limit, clocks.sm, clocks.max.sm: {info['nvidia_smi']}")
    print(f"lib {info['lib']} | median over {len(recs)} steps (after {a.warmup} warm-up)")
    for k in keys:
        n = sum(1 for rec in recs if k in rec)
        unit = "us" if k.startswith("step_us") else ("ns" if k.startswith(("span", "gap", "step end")) else "cycles")
        print(f"  {k:<48s} {med[k]:>10.1f} {unit}" + ("" if n == len(recs) else f"   ({n} steps)"))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"info": info, "steps": len(recs), "median": med}, f, indent=1)


if __name__ == "__main__":
    main()
