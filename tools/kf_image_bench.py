"""Times the keyframe image (liliom_kf_export / liliom_kf_import) of a 300-keyframe Horizon store with ~20k-point full clouds,
with and without the full clouds, against replaying the store's kf_add + kf_add_full calls, and splits one export and one import
into the checksum kernel (k_kf_image) and the PCIe copies with torch.profiler.  The caller's image buffer is pageable (what
Context.kf_export / kf_import use) or pinned (a caller that keeps one pinned buffer).  Prints the card's name and power limit.

    python tools/kf_image_bench.py [--kf 300] [--reps 7]"""
from __future__ import annotations

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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kf", type=int, default=300)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    import liliom_b200 as L
    from liliom_b200 import synth
    lib = L._binding.lib()
    bp = L.backend_default_params(0)
    seq = synth.make_keyframe_sequence(a.kf, stride=48, seed=5, full=True)
    A = L.Context(variant=0)
    for e, s, _, f in seq:
        kid, _, _ = A.kf_add(bp, e, s, download=False)
        A.kf_add_full(bp, kid, f)
    D = L.Context(variant=0)
    res = {"card": card(), "keyframes": a.kf, "full_points": int(sum(len(f) for *_, f in seq))}

    def med(f):
        f()                                          # warm-up: every buffer at its size
        t = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            f()
            t.append(time.perf_counter() - t0)
        return 1e3 * float(np.median(t)), 1e3 * float(min(t))

    for full in (True, False):
        flags = 1 if full else 0
        n = C.c_longlong()
        assert lib.liliom_kf_export(A._h, None, 0, flags, None, 0, C.byref(n)) == 0
        size = n.value
        page = np.empty(size, np.uint8)
        pin = torch.empty(size, dtype=torch.uint8, pin_memory=True)
        tag = "full" if full else "scan"
        res[f"{tag}_bytes"] = size
        for kind, ptr in (("pageable", page.ctypes.data), ("pinned", pin.data_ptr())):
            def export(ptr=ptr):
                assert lib.liliom_kf_export(A._h, None, 0, flags, C.c_void_p(ptr), size, C.byref(n)) == 0

            def imp(ptr=ptr):
                D.kf_clear()
                f, k = C.c_int(), C.c_int()
                assert lib.liliom_kf_import(D._h, C.c_void_p(ptr), size, C.byref(f), C.byref(k)) == 0
            res[f"{tag}_export_{kind}_ms"] = med(export)
            res[f"{tag}_import_{kind}_ms"] = med(imp)
            if kind == "pinned":
                assert bytes(pin.numpy()) == bytes(page)
            assert D.kf_export(full=full) == bytes(page)

        def replay(full=full):
            R = L.Context(variant=0)
            for e, s, _, f in seq:
                kid, _, _ = R.kf_add(bp, e, s, download=False)
                if full:
                    R.kf_add_full(bp, kid, f)
            R.close()
        res[f"{tag}_replay_ms"] = med(replay)

        # one export and one import (pinned) under the profiler: the checksum kernel against the copies
        from torch.profiler import ProfilerActivity, profile
        ptr = pin.data_ptr()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            assert lib.liliom_kf_export(A._h, None, 0, flags, C.c_void_p(ptr), size, C.byref(n)) == 0
            torch.cuda.synchronize()
            D.kf_clear()
            f_, k_ = C.c_int(), C.c_int()
            assert lib.liliom_kf_import(D._h, C.c_void_p(ptr), size, C.byref(f_), C.byref(k_)) == 0
            torch.cuda.synchronize()
        kern, copy = [], []
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            us = ev.time_range.elapsed_us()
            if "k_kf_image" in ev.name:
                kern.append(us)
            elif "Memcpy" in ev.name and (ev.name.find("DtoH") >= 0 or ev.name.find("HtoD") >= 0):
                copy.append((ev.name, us))
        res[f"{tag}_kernel_us"] = kern
        res[f"{tag}_big_copies_us"] = sorted([c for c in copy if c[1] > 100], key=lambda c: -c[1])[:4]
    print(json.dumps(res))
    A.close(); D.close()


if __name__ == "__main__":
    main()
