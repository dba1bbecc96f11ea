"""TEST INFRASTRUCTURE: the library's calls as a catalogue of operations, for the history tests (tests/test_gpu_history.py).

A context keeps grow-only scratch, control words and per-call state between calls, and each call has to rewrite whatever it
reads.  The history tests run every operation here after other calls and compare it with the same operation on a fresh context.

An operation (Op) has a name, the context kinds it runs on (KINDS) and named inputs.  An input is a callable op(ctx) that runs the
call on the context, installing first whatever context state it needs (the map, the keyframe store, the resident sweep, the
ring and time sources), so that its outputs depend on the call's own arguments alone, and returns everything observable as a
dict of bytes: the returned clouds, poses, stats rows, counts and status codes, and the state the next call reads (the resident
clouds, the filtered map, the stored keyframes).  A refused call returns its error code.  `nxt(ctx)` is the call that follows the
operation in a real process (the next scan, the next map update, the next keyframe), reading the state the operation left.

Input names: "large", "small", "empty", "refused", and "n<k>" for a size just either side of a launch's block size.  The inputs
come from the suite's generators (synth, vg_adversarial, bk_adversarial, hz_adversarial's Livox records), sliced to size.

s2m: the operation runs a scan-to-map step.  dev_count: that step's query count is known only on the device, so its launch is
sized from the previous step's query count (s2m_plan's n_last) and the comparison replays the history's last s2m input first."""
from __future__ import annotations

import ctypes as C
import functools
import os
from dataclasses import dataclass, field
from typing import Callable

import numpy as np

import bk_adversarial as BK
import vg_adversarial as VG

KINDS = {"48": dict(variant=0), "32": dict(variant=1), "48chain": dict(variant=0, env={"LILIOM_HZ_CHAIN": "1"})}
BLOCK_EDGES = (1, 127, 128, 129, 255, 256, 257, 511, 512, 513)
IDENT7 = np.array([1.0, 0, 0, 0, 0, 0, 0])
IDENT_Q = (1.0, 0.0, 0.0, 0.0)
TINY_LEAF = 1e-4          # PCL declines every keyframe-sized cloud at this leaf: global_map gives the stored cloud back
ITERS = 4
ALL = 1 << 30             # a slice bound past every input: the whole cloud


def _L():
    import liliom_b200 as L
    return L


def b(a) -> bytes:
    if isinstance(a, (bytes, bytearray)):
        return bytes(a)
    if isinstance(a, C.Array) or isinstance(a, C.Structure):
        return C.string_at(C.addressof(a), C.sizeof(a))
    if isinstance(a, list):
        return b"".join(b(x) for x in a)
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def code(f) -> int:
    """f()'s error code (0: it ran)"""
    L = _L()
    try:
        f()
        return 0
    except L.LiliomError as e:
        return e.code


def make_ctx(kind: str, **params):
    L = _L()
    k = KINDS[kind]
    p = L.default_params(k["variant"])
    for n, v in params.items():
        setattr(p, n, v)
    env = k.get("env", {})
    old = {n: os.environ.get(n) for n in env}
    os.environ.update(env)
    try:
        return L.Context(p)
    finally:
        for n, v in old.items():
            if v is None:
                os.environ.pop(n, None)
            else:
                os.environ[n] = v


def stride(kind: str) -> int:
    return 48 if KINDS[kind]["variant"] == 0 else 32


@dataclass
class Op:
    name: str
    kinds: tuple
    inputs: dict                      # input name -> op(ctx) -> dict of bytes
    nxt: Callable                     # the following call: nxt(ctx) -> dict of bytes
    s2m: bool = False
    dev_count: bool = False
    oracle: dict = field(default_factory=dict)   # input name -> () -> dict of bytes, a subset of the input's outputs
    refused_pure: bool = True         # the refused input installs no state of its own before the call is refused


# ------------------------------------------------------------------------------------------------------------- inputs
@functools.lru_cache(None)
def world():
    """The suite's synthetic world: the 100k-point map, a Horizon sweep (PT48) and an HDL-64E sweep (PT32, ~130k points, with
    each return's ring) from the default pose, a perturbed guess, a short HDL sweep and a keyframe sequence of both strides."""
    from liliom_b200 import synth
    m, _ = synth.make_map(100_000)
    T = synth.default_true_pose()
    hz, q_hz = synth.make_horizon_sweep(T)
    hdl, q_hdl, ring, step = synth.make_hdl64_sweep(T, grid=True)
    hdl_s, _, ring_s, step_s = synth.make_hdl64_sweep(T, seed=5, steps=128, grid=True)
    kf = {48: synth.make_keyframe_sequence(12, 48, full=True), 32: synth.make_keyframe_sequence(12, 32, full=True)}
    return dict(map=m, T=T, guess=synth.perturbed_pose(T), hz=hz, q_hz=q_hz, hdl=hdl, q_hdl=q_hdl, ring=ring, step=step,
                hdl_s=hdl_s, ring_s=ring_s, step_s=step_s, kf=kf)


def sweep(kind):
    """(points, q_imu) of the kind's extractor: the Horizon sweep (48) or the HDL-64E sweep (32)"""
    w = world()
    return (w["hz"], w["q_hz"]) if stride(kind) == 48 else (w["hdl"], w["q_hdl"])


def as_stride(pts, s):
    return pts if pts.dtype.itemsize == s else VG.to32(pts)


def sizes(large_n, small_n):
    """{input name: point count}: large, small, empty and the block edges"""
    out = {"large": large_n, "small": small_n, "empty": 0}
    out.update({f"n{k}": k for k in BLOCK_EDGES})
    return out


@functools.lru_cache(None)
def livox(stride_bytes):
    """The Horizon sweep as Livox CustomPoint records, in time order (20-byte records or the 19-byte wire layout)"""
    from test_gpu_kf_handoff import _livox
    r = _livox(world()["hz"])
    if stride_bytes == 20:
        return r
    return np.ascontiguousarray(r).view(np.uint8).reshape(len(r), 20)[:, :19].copy().reshape(-1)


def livox_first(stride_bytes, n):
    r = livox(stride_bytes)
    return r[:n] if stride_bytes == 20 else r[:19 * n]


@functools.lru_cache(None)
def pc2(layout, big):
    """The HDL-64E sweep (big) or a 128-column one as the PointCloud2 of a driver layout (synth.encode_pc2)"""
    from liliom_b200 import synth
    w = world()
    if big:
        return synth.encode_pc2(w["hdl"], w["ring"], w["step"], layout)
    return synth.encode_pc2(w["hdl_s"], w["ring_s"], w["step_s"], layout, steps=128)


def pc2_first(n):
    """the first n returns of the HDL-64E sweep as a pcl32 message (one row)"""
    from liliom_b200 import synth
    w = world()
    return synth.encode_pc2(w["hdl"][:n], w["ring"][:n], w["step"][:n], "pcl32")


# ---------------------------------------------------------------------------------------------------------- the ops
def _sources(c):
    L = _L()
    if c.stride == 32:
        c.set_ring_source(L.RING_ELEVATION)
        c.set_time_source(L.TIME_AZIMUTH)


def feats_state(c):
    """the clouds the last extraction left resident (or the refusal code)"""
    L = _L()
    try:
        s, e, k = c.features_download()
        return {"res_surf": b(s), "res_edge": b(e), "res_cut": b(k)}
    except L.LiliomError as e:
        return {"res": e.code}


def _extract_out(r):
    return {"surf": b(r[0]), "edge": b(r[1]), "cut": b(r[2])}


def nxt_extract(c):
    """publishCloudLast's de-skew on the resident clouds, then the keyframe hand-off to this context's own store"""
    L = _L()
    out = {"undistort": code(lambda: c.undistort_resident((0.31, -0.12, 0.05), (0.9999, 0.01, -0.005, 0.002)))}
    out.update(feats_state(c))
    c.kf_clear()
    bp = L.backend_default_params(0 if c.stride == 48 else 1)
    out["kf"] = code(lambda: out.__setitem__("kfr", repr(c.kf_add_resident(bp, c))))
    if out["kf"] == 0:
        out["kf_full"] = b(c.global_map(L.KF_FULL, [0], [IDENT7], TINY_LEAF))
    return out


def nxt_resident_sweep(c):
    """the extraction of the sweep a decode left resident"""
    _sources(c)
    q = world()["q_hz"] if c.stride == 48 else world()["q_hdl"]
    out = {}
    out["rc"] = code(lambda: out.__setitem__("n", repr(c.extract_resident(q))))
    out.update(feats_state(c))
    return out


def nxt_vg(c):
    cloud = as_stride(VG.heavy(0.4), c.stride)
    return {"vg_next": b(c.voxelgrid(cloud, 0.4))}


def s2m_feats(n):
    """n body-frame queries (float4) of the Horizon sweep"""
    hz = world()["hz"]
    n = min(n, len(hz))
    f = np.ones((n, 4), np.float32)
    f[:, 0], f[:, 1], f[:, 2] = hz["x"][:n], hz["y"][:n], hz["z"][:n]
    return f


def nxt_s2m(c):
    """the next scan: a host-count GN step of 300 queries on the installed map"""
    w = world()
    out = {}
    out["rc"] = code(lambda: out.__setitem__("pose", b(c.scan_to_map(s2m_feats(300)[::-1].copy(), w["guess"], ITERS, mode=_L().MODE_GN)[0])))
    return out


def _s2m_out(pose, stats):
    return {"pose": b(pose), "stats": b(stats) if stats is not None else b""}


def nxt_map(c):
    """the next map update (a 2000-point scan) and the map it leaves"""
    w = world()
    pts = as_stride(w["hz"][5000:7000], c.stride)
    out = {"n": c.map_update(pts, w["T"])}
    out.update(map_state(c))
    return out


def map_state(c):
    L = _L()
    out = {"map": b(c.map_download())}
    try:
        out["map_cloud"] = b(c.map_download_cloud())
    except L.LiliomError as e:
        out["map_cloud"] = e.code
    return out


def kf_seq(c, k):
    return world()["kf"][c.stride][:k]


def store(c, k, full=False):
    """kf_clear, then the first k keyframes of the sequence (their full clouds too)"""
    L = _L()
    bp = L.backend_default_params(0 if c.stride == 48 else 1)
    c.kf_clear()
    out = []
    for e, s, _p, f in kf_seq(c, k):
        kid, eds, sds = c.kf_add(bp, e, s)
        out += [kid, b(eds), b(sds)]
        if full:
            out.append(c.kf_add_full(bp, kid, f))
    return bp, out


def store_state(c):
    L = _L()
    n = c.kf_count()
    ids = list(range(n))
    return {"kf_n": n, "kf_surf": b(c.global_map(L.KF_SURF, ids, [IDENT7] * n, TINY_LEAF)) if n else b""}


def nxt_kf(c):
    """the next keyframe, and the local map of the whole store"""
    L = _L()
    bp = L.backend_default_params(0 if c.stride == 48 else 1)
    e, s, _p, _f = world()["kf"][c.stride][11]
    kid, eds, sds = c.kf_add(bp, e, s)
    n = c.kf_count()
    poses = [p for _e, _s, p, _f in kf_seq(c, 11)][:n - 1] + [_p]
    return {"kid": kid, "eds": b(eds), "sds": b(sds), "bmap": repr(c.bmap_build(bp, list(range(n)), poses)),
            "l0": b(c.bmap_download(0)), "l1": b(c.bmap_download(1))}


def _helper(c):
    """the second session of a batched call: a fresh context of c's stride"""
    return make_ctx("48" if c.stride == 48 else "32")


def _ops_decode():
    L = _L()
    ops = []
    for sb in (20, 19):
        def run(n, sb=sb):
            return lambda c: {"cloud": b(c.convert_livox(livox_first(sb, n), stride=sb))}
        inputs = {k: run(n) for k, n in sizes(ALL, 300).items()}
        inputs["refused"] = lambda c: {"rc": L._binding.lib().liliom_convert_livox(c._h, None, 5, 20, None, 0)}
        ops.append(Op(f"convert_livox{sb}", ("48",), inputs, nxt_resident_sweep,
                      oracle={"large": lambda sb=sb: {"cloud": b(_oracle().convert_livox(livox(sb), sb))}}))
    from test_wire_host import LAYOUTS
    for layout in LAYOUTS:
        def run(msg_f, layout=layout):
            return lambda c: (_sources(c), {"cloud": b(c.convert_pc2(msg_f()))})[1]
        inputs = {"large": run(lambda layout=layout: pc2(layout, True)), "small": run(lambda layout=layout: pc2(layout, False))}
        if layout == "pcl32":
            inputs.update({k: run(lambda n=n: pc2_first(n)) for k, n in sizes(0, 0).items() if k not in ("large", "small")})

        inputs["refused"] = lambda c: {"rc": code(lambda: c.convert_pc2(L.PC2(b"", 1, 5, 16, 80, [])))}   # no x, y, z fields
        ops.append(Op(f"convert_pc2_{layout}", ("32",), inputs, nxt_resident_sweep))

    def batch(msgs_f, refused=False):
        def f(c):
            _sources(c)
            h = _helper(c)
            try:
                clouds, st = L.convert_batch([c, h], msgs_f(c), download=True)
                if refused:                # session 0 refused: only the statuses are this call's
                    return {"st": b(st)}
                return {"clouds": b([x for x in clouds if x is not None]), "st": b(st)}
            finally:
                h.close()
        return f

    def msgs(c, n):
        if c.stride == 48:
            return [livox_first(20, n), livox_first(20, 40)]
        return [pc2_first(n), pc2_first(40)]

    inputs = {k: batch(lambda c, n=n: msgs(c, n)) for k, n in sizes(24_000, 300).items()}
    inputs["refused"] = batch(lambda c: [(livox_first(20, 10).view(np.uint8), 21), livox_first(20, 40)] if c.stride == 48
                              else [L.PC2(b"", 1, 5, 16, 80, []), pc2_first(40)], refused=True)
    ops.append(Op("convert_batch", ("48", "32"), inputs, nxt_resident_sweep))
    return ops


def _oracle():
    import oracle_lib
    return oracle_lib


def _ops_extract():
    L = _L()
    ops = []

    def hz_run(n):
        def f(c):
            pts, q = sweep("48")
            return {**_extract_out(c.extract_horizon(pts[:n], q)), **feats_state(c)}
        return f

    def hz_oracle(n):
        pts, q = sweep("48")
        return lambda: _extract_out(_oracle().extract_horizon(pts[:n], q))

    inputs = {k: hz_run(n) for k, n in sizes(ALL, 2000).items()}
    inputs["refused"] = lambda c: {"rc": code(lambda: c.extract_rot(world()["hdl"][:100], world()["q_hdl"])), **feats_state(c)}
    ops.append(Op("extract_horizon", ("48", "48chain"), inputs, nxt_extract,
                  oracle={"large": hz_oracle(ALL), "small": hz_oracle(2000)}))

    def hzl_run(sb, n):
        return lambda c: {**_extract_out(c.extract_horizon_livox(livox_first(sb, n), world()["q_hz"], stride=sb)), **feats_state(c)}
    inputs = {k: hzl_run(20, n) for k, n in sizes(ALL, 2000).items()}
    inputs["s19"] = hzl_run(19, ALL)
    inputs["refused"] = lambda c: {"rc": L._binding.lib().liliom_extract_horizon_livox(c._h, None, 4, 20, None, None, 0, None, None, 0,
                                                                                          None, None, 0, None)}
    ops.append(Op("extract_horizon_livox", ("48", "48chain"), inputs, nxt_extract))

    def rot_run(n):
        def f(c):
            _sources(c)
            pts, q = sweep("32")
            return {**_extract_out(c.extract_rot(pts[:n], q)), **feats_state(c)}
        return f

    def rot_oracle(n):
        pts, q = sweep("32")
        p = L.default_params(1)
        return lambda: _extract_out(_oracle().extract_rot(pts[:n], q, line_num=p.line_num, ds_rate=p.ds_rate)[1:4])

    inputs = {k: rot_run(n) for k, n in sizes(ALL, 8000).items()}
    inputs["refused"] = lambda c: (c.set_ring_source(L.RING_FIELD), {"rc": code(lambda: c.extract_rot(world()["hdl"][:100], world()["q_hdl"])),
                                                                    **feats_state(c)})[1]
    ops.append(Op("extract_rot", ("32",), inputs, nxt_extract, oracle={"small": rot_oracle(8000)}, refused_pure=False))

    def rotpc2_run(msg_f):
        return lambda c: (_sources(c), {**_extract_out(c.extract_rot_pc2(msg_f(), world()["q_hdl"])), **feats_state(c)})[1]
    inputs = {"large": rotpc2_run(lambda: pc2("pcl32", True)), "small": rotpc2_run(lambda: pc2("ouster48", False)),
              "empty": rotpc2_run(lambda: pc2_first(0)), "n257": rotpc2_run(lambda: pc2_first(257))}
    ops.append(Op("extract_rot_pc2", ("32",), inputs, nxt_extract))

    def res_run(n):
        def f(c):
            _sources(c)
            pts, q = sweep(stride_kind(c))
            c.upload_scan(pts[:n])
            return {"n": repr(c.extract_resident(q)), **feats_state(c)}
        return f
    inputs = {k: res_run(n) for k, n in sizes(ALL, 2000).items()}
    ops.append(Op("extract_resident", ("48", "48chain", "32"), inputs, nxt_extract))

    def resb_run(n):
        def f(c):
            _sources(c)
            pts, q = sweep(stride_kind(c))
            h = _helper(c)
            try:
                c.upload_scan(pts[:n]); h.upload_scan(pts[:700])
                cnt, st = L.extract_resident_batch([c, h], np.stack([q, q]))
                return {"n": b(cnt), "st": b(st), **feats_state(c)}
            finally:
                h.close()
        return f
    inputs = {k: resb_run(n) for k, n in sizes(24_000, 2000).items()}
    ops.append(Op("extract_resident_batch", ("48", "32"), inputs, nxt_extract))

    def und_run(n):
        def f(c):
            pts, _ = sweep(stride_kind(c))
            return {"out": b(c.undistort(pts[:n], (0.3, -0.1, 0.05), (0.9999, 0.01, -0.005, 0.002)))}
        return f
    inputs = {k: und_run(n) for k, n in sizes(24_000, 2000).items()}
    inputs["refused"] = lambda c: {"rc": L._binding.lib().liliom_undistort(c._h, None, 3, None, None)}
    ops.append(Op("undistort", ("48", "32"), inputs, nxt_vg))

    def undr_run(n):
        def f(c):
            _sources(c)
            pts, q = sweep(stride_kind(c))
            c.upload_scan(pts[:n])
            c.extract_resident(q)
            return {"rc": code(lambda: c.undistort_resident((0.3, -0.1, 0.05))), **feats_state(c)}
        return f
    inputs = {k: undr_run(n) for k, n in sizes(24_000, 2000).items()}
    ops.append(Op("undistort_resident", ("48", "32"), inputs, nxt_extract))
    return ops


def stride_kind(c):
    return "48" if c.stride == 48 else "32"


def _ops_vg():
    L = _L()

    def run(cloud_f, leaf=0.4):
        return lambda c: {"vg": b(c.voxelgrid(as_stride(cloud_f(), c.stride), leaf))}
    inputs = {"large": run(lambda: VG.sized(60_000, 0.4)), "coop": run(lambda: VG.sized(VG.VGC_NCAP, 0.4)),
              "sort": run(lambda: VG.sized(VG.VGC_NCAP + 1, 0.4)), "small": run(lambda: VG.heavy(0.4)),
              "payload": run(lambda: VG.payload(0.4))}
    inputs.update({k: run(lambda n=n: VG.sized(600, 0.4)[:n]) for k, n in sizes(0, 0).items() if k not in ("large", "small")})
    inputs["refused"] = lambda c: {"rc": code(lambda: c.voxelgrid(as_stride(VG.heavy(0.4), c.stride), 0.0))}
    oracle = {"coop": lambda: {"vg": b(_oracle().voxelgrid(VG.sized(VG.VGC_NCAP, 0.4), 0.4))},
              "large": lambda: {"vg": b(_oracle().voxelgrid(VG.sized(60_000, 0.4), 0.4))}}
    return [Op("voxelgrid", ("48", "32"), inputs, nxt_vg, oracle=oracle)]


def _ops_s2m():
    L = _L()
    w = world()
    ops = []
    for mode, mname in ((L.MODE_GN, "gn"), (L.MODE_CERES, "ceres")):
        cnt = ITERS if mode == L.MODE_GN else 2

        def run(n, mode=mode, cnt=cnt):
            def f(c):
                c.map_set_points(w["map"])
                pose, st = c.scan_to_map(s2m_feats(n), w["guess"], cnt, 6, mode)
                return _s2m_out(pose, st)
            return f
        inputs = {k: run(n) for k, n in sizes(24_000, 200).items()}
        inputs["mid"] = run(3000)

        def refused(c, mode=mode, cnt=cnt):
            c.map_set_points(w["map"][:5])
            return {"rc": code(lambda: c.scan_to_map(s2m_feats(200), w["guess"], cnt, 6, mode))}
        inputs["refused"] = refused
        ops.append(Op(f"scan_to_map_{mname}", ("48", "32"), inputs, nxt_s2m, s2m=True, refused_pure=False))

        def res_run(n, mode=mode, cnt=cnt):
            def f(c):
                c.map_set_points(w["map"])
                c.upload_feats(s2m_feats(n))
                pose, st = c.scan_to_map_resident(w["guess"], cnt, 6, mode, want_stats=True)
                return _s2m_out(pose, st)
            return f
        inputs = {k: res_run(n) for k, n in sizes(24_000, 200).items() if k != "empty"}
        inputs["mid"] = res_run(3000)
        ops.append(Op(f"scan_to_map_resident_{mname}", ("48", "32"), inputs, nxt_s2m, s2m=True))

        def odo_run(n, mode=mode, cnt=cnt):
            def f(c):
                pts, _ = sweep(stride_kind(c))
                c.map_clear()
                c.map_set_points(w["map"])
                pose, st, ds = c.odometry(pts[:n], w["guess"], cnt, 6, mode)
                return {**_s2m_out(pose, st), "ds": b(ds)}
            return f
        inputs = {k: odo_run(n) for k, n in sizes(24_000, 1500).items()}
        inputs["mid"] = odo_run(8000)
        inputs["refused"] = lambda c, mode=mode, cnt=cnt: (c.map_set_points(w["map"][:5]),
                                                          {"rc": code(lambda: c.odometry(sweep(stride_kind(c))[0][:500], w["guess"], cnt, 6, mode))})[1]
        ops.append(Op(f"odometry_{mname}", ("48", "32"), inputs, nxt_map, s2m=True, dev_count=True, refused_pure=False))

        def odor_run(n, mode=mode, cnt=cnt):
            def f(c):
                _sources(c)
                pts, q = sweep(stride_kind(c))
                c.map_clear()
                c.map_set_points(w["map"])
                c.upload_scan(pts[:n])
                c.extract_resident(q)
                pose, st, ds = c.odometry_resident(w["guess"], cnt, 6, mode, want_ds=True, cap=65536)
                return {**_s2m_out(pose, st), "ds": b(ds)}
            return f
        inputs = {"large": odor_run(ALL), "small": odor_run(3000), "n513": odor_run(513)}
        ops.append(Op(f"odometry_resident_{mname}", ("48", "32"), inputs, nxt_map, s2m=True, dev_count=True))

        def batch_run(n, odo, mode=mode, cnt=cnt):
            def f(c):
                h = _helper(c)
                try:
                    for x, m in ((c, n), (h, 700)):
                        x.map_clear()
                        x.map_set_points(w["map"])
                        if odo:
                            _sources(x)
                            pts, q = sweep(stride_kind(x))
                            x.upload_scan(pts[:m]); x.extract_resident(q)
                        else:
                            x.upload_feats(s2m_feats(m))
                    poses = [w["guess"], w["guess"]]
                    if odo:
                        r = L.odometry_resident_batch_ex([c, h], poses, cnt, 6, mode, want_stats=True, want_ds=True)
                        return {"pose": b(r[0][0]), "st": b(r[1]), "stats": b(r[2][0]), "ds": b(r[3][0])}
                    r = L.scan_to_map_resident_batch_ex([c, h], poses, cnt, 6, mode, want_stats=True)
                    return {"pose": b(r[0][0]), "st": b(r[1]), "stats": b(r[2][0])}
                finally:
                    h.close()
            return f
        for odo in (False, True):
            nm = ("odometry" if odo else "scan_to_map") + f"_resident_batch_{mname}"
            inputs = {"large": batch_run(24_000, odo), "mid": batch_run(3000, odo), "small": batch_run(200 if not odo else 1500, odo),
                      "n129": batch_run(129, odo)}
            ops.append(Op(nm, ("48", "32"), inputs, nxt_map if odo else nxt_s2m, s2m=True, dev_count=odo))
    return ops


def _ops_map():
    L = _L()
    w = world()
    ops = []

    def upd_run(k, n):
        """map_clear, then k map updates of n-point scans along the path"""
        def f(c):
            c.map_clear()
            pts = as_stride(w["hz"], c.stride)
            ns = []
            for i in range(k):
                p = np.array(w["T"]); p[4] += 0.3 * i
                ns.append(c.map_update(pts[(i * 997) % 4000:][:n], p))
            return {"ns": repr(ns), **map_state(c)}
        return f
    inputs = {"large": upd_run(14, 20_000), "small": upd_run(2, 300), "empty": upd_run(3, 0), "n257": upd_run(4, 257)}
    inputs["refused"] = lambda c: {"rc": L._binding.lib().liliom_map_update(c._h, None, 4, None, None), **map_state(c)}
    ops.append(Op("map_update", ("48", "32"), inputs, nxt_map))

    def push_run(k, n):
        def f(c):
            c.map_clear()
            pts = as_stride(w["hz"], c.stride)
            for i in range(k):
                p = np.array(w["T"]); p[5] += 0.2 * i
                c.map_push_frame(pts[(i * 613) % 4000:][:n], p)
            return {"m": c.map_rebuild(), **map_state(c)}
        return f
    inputs = {"large": push_run(12, 20_000), "small": push_run(1, 300), "empty": push_run(1, 0), "n511": push_run(2, 511)}
    ops.append(Op("map_push_rebuild", ("48", "32"), inputs, nxt_map))

    def clear_run(k, n):
        def f(c):
            upd_run(k, n)(c)
            c.map_clear()
            return map_state(c)
        return f
    ops.append(Op("map_clear", ("48", "32"), {"large": clear_run(14, 20_000), "small": clear_run(2, 300)}, nxt_map))

    def set_run(n, cloud):
        def f(c):
            if cloud:
                c.map_set_cloud(as_stride(w["hz"][:n], c.stride))
            else:
                c.map_set_points(w["map"][:n])
            return {**map_state(c), **nxt_s2m(c)}
        return f
    inputs = {"large": set_run(100_000, False), "small": set_run(500, False), "cloud": set_run(20_000, True), "n129": set_run(129, False)}
    inputs["refused"] = lambda c: {"rc": L._binding.lib().liliom_map_set_points(c._h, None, 3)}
    ops.append(Op("map_set", ("48", "32"), inputs, nxt_s2m, s2m=True))

    def updr_run(n, batch):
        def f(c):
            _sources(c)
            c.map_clear()
            pts, q = sweep(stride_kind(c))
            c.map_update(as_stride(w["hz"][:3000], c.stride), w["T"])
            c.upload_scan(pts[:n]); c.extract_resident(q)
            c.odometry_resident(w["guess"], 1, 6, L.MODE_GN, want_stats=False)
            if batch:
                h = _helper(c)
                try:
                    h.map_update(as_stride(w["hz"][:800], h.stride), w["T"])
                    h.upload_scan(pts[:900]); h.extract_resident(q)
                    h.odometry_resident(w["guess"], 1, 6, L.MODE_GN, want_stats=False)
                    nm, st = L.map_update_batch([c, h], np.stack([w["T"], w["T"]]))
                    return {"n": b(nm), "st": b(st), **map_state(c)}
                finally:
                    h.close()
            return {"n": c.map_update_resident(w["T"]), **map_state(c)}
        return f
    for batch in (False, True):
        inputs = {"large": updr_run(ALL, batch), "small": updr_run(1500, batch), "n257": updr_run(257, batch)}
        ops.append(Op("map_update_batch" if batch else "map_update_resident", ("48", "32"), inputs, nxt_map, s2m=True, dev_count=True))
    return ops


def _ops_backend():
    L = _L()
    ops = []

    def kf_run(k, full=False):
        def f(c):
            _bp, out = store(c, k, full)
            return {"kfs": b(b"".join(x if isinstance(x, bytes) else repr(x).encode() for x in out)), **store_state(c)}
        return f
    inputs = {"large": kf_run(10), "small": kf_run(2), "empty": kf_run(0)}
    inputs["refused"] = lambda c: {"rc": L._binding.lib().liliom_kf_add(c._h, None, None, 0, None, 0, None, None, 0, None, None, 0, None),
                                   **store_state(c)}
    ops.append(Op("kf_add", ("48", "32"), inputs, nxt_kf))
    ops.append(Op("kf_add_full", ("48", "32"), {"large": kf_run(10, True), "small": kf_run(2, True)}, nxt_kf))

    def kfr_run(n):
        def f(c):
            _sources(c)
            bp = L.backend_default_params(0 if c.stride == 48 else 1)
            c.kf_clear()
            pts, q = sweep(stride_kind(c))
            c.upload_scan(pts[:n]); c.extract_resident(q)
            return {"r": repr(c.kf_add_resident(bp, c)), **store_state(c),
                    "full": b(c.global_map(L.KF_FULL, [0], [IDENT7], TINY_LEAF))}
        return f
    ops.append(Op("kf_add_resident", ("48", "32"), {"large": kfr_run(ALL), "small": kfr_run(1500), "n129": kfr_run(129)}, nxt_kf))

    def bmap_run(k, kw):
        """store k keyframes, build the local map of them, then the window correspondences and blocks of kw of them"""
        def f(c):
            bp, _ = store(c, k)
            seq = kf_seq(c, k)
            poses = [p for _e, _s, p, _f in seq]
            out = {"bmap": repr(c.bmap_build(bp, list(range(k)), poses)), "l0": b(c.bmap_download(0)), "l1": b(c.bmap_download(1))}
            if kw:
                win = list(range(k - kw, k))
                ne, ns = c.backend_window_correspond(bp, win, [poses[i] for i in win])
                out.update(ne=b(ne), ns=b(ns), blocks=b(c.backend_window_blocks([poses[i] for i in win])))
                out["corr"] = b([b(x) for s in range(kw) for kind in (0, 1) for x in c.backend_window_corr(s, kind)])
            return out
        return f
    inputs = {"large": bmap_run(10, 6), "small": bmap_run(2, 1), "nowin": bmap_run(3, 0)}
    inputs["refused"] = lambda c: (store(c, 2), {"rc": code(lambda: c.backend_window_blocks([IDENT7] * 3))})[1]
    ops.append(Op("bmap_window", ("48", "32"), inputs, nxt_kf, refused_pure=False))

    def winb_run(k, kw):
        def f(c):
            h = _helper(c)
            try:
                out = {}
                win_ids, win_poses, bps = [], [], []
                for x, kk, ww in ((c, k, kw), (h, 3, 2)):
                    bp, _ = store(x, kk)
                    poses = [p for _e, _s, p, _f in kf_seq(x, kk)]
                    x.bmap_build(bp, list(range(kk)), poses)
                    win = list(range(kk - ww, kk))
                    win_ids.append(win); win_poses.append([poses[i] for i in win]); bps.append(bp)
                r, st = L.backend_window_correspond_batch([c, h], bps, win_ids, win_poses)
                blk, st2 = L.backend_window_blocks_batch([c, h], win_poses)
                out.update(ne=b(r[0][0]), ns=b(r[0][1]), st=b(st), blocks=b(blk[0]), st2=b(st2))
                out["corr"] = b([b(x) for s in range(kw) for kind in (0, 1) for x in c.backend_window_corr(s, kind)])
                return out
            finally:
                h.close()
        return f
    ops.append(Op("backend_window_batch", ("48", "32"), {"large": winb_run(10, 6), "small": winb_run(2, 1)}, nxt_kf))

    def loop_run(k, batch):
        def f(c):
            store(c, k, full=False)
            poses = [p for _e, _s, p, _f in kf_seq(c, k)]
            src, tgt = [k - 1], list(range(k - 1))
            args = (src, [poses[-1]], tgt, poses[:-1])
            if not batch:
                r = c.loop_align(*args, 0.4, max_iter=20)
            else:
                h = _helper(c)
                try:
                    store(h, 3)
                    hp = [p for _e, _s, p, _f in kf_seq(h, 3)]
                    rr, st = L.loop_align_batch([c, h], [src, [2]], [[poses[-1]], [hp[2]]], [tgt, [0, 1]], [poses[:-1], hp[:2]],
                                                [dict(leaf=0.4, max_iter=20)] * 2)
                    r = rr[0]
                finally:
                    h.close()
            return {"T": b(r[0]), "rest": repr(r[1:]), "kfc": b(c.kf_cloud(src, [poses[-1]], 0.4)),
                    "gm": b(c.global_map(L.KF_SURF, tgt, poses[:-1], 0.4))}
        return f
    for batch in (False, True):
        inputs = {"large": loop_run(10, batch), "small": loop_run(2, batch)}
        if not batch:
            inputs["refused"] = lambda c: (store(c, 2), {"rc": code(lambda: c.loop_align([0], [IDENT7], [1], [IDENT7], 0.0))})[1]
        ops.append(Op("loop_align_batch" if batch else "loop_align", ("48", "32"), inputs, nxt_kf, refused_pure=False))

    def icp_run(n_src, n_tgt):
        def f(c):
            e, s, p, full = kf_seq(c, 2)[1]
            tgt = BK.f4(np.ascontiguousarray(kf_seq(c, 1)[0][3])[:n_tgt]) if n_tgt else np.zeros((0, 4), np.float32)
            src = BK.f4(np.ascontiguousarray(full)[:n_src]) if n_src else np.zeros((0, 4), np.float32)
            T, fit, conv, it = c.icp_align(src, tgt, max_iter=15)
            return {"T": b(T), "rest": repr((fit, conv, it))}
        return f
    inputs = {"large": icp_run(20_000, 20_000), "small": icp_run(300, 4000), "empty": icp_run(0, 4000)}
    inputs.update({f"n{k}": icp_run(k, 4000) for k in (255, 256, 257)})
    ops.append(Op("icp_align", ("48", "32"), inputs, nxt_s2m))

    def corr_run(kind, n):
        def f(c):
            W = BK.backend_world("far")
            variant = 0 if c.stride == 48 else 1
            body = np.array(W["pose"])
            if kind == "edge":
                c.map_set_points(W["edge_map"])
                q = BK.f4(W["edge_q"])[:n]
                v, pa, pb = c.correspond_edge(q, W["pose"], variant)
                return {"v": b(v), "pa": b(pa), "pb": b(pb), "blk": b(c.backend_edge_block(body, 0.6, 1.0))}
            if kind == "refl":
                c.map_set_cloud(W["surf_map"])
                v, pl, sc = c.correspond_surf_refl(W["surf_q"][:n], W["pose"], 1.0, BK.SURF_DIST_THRES, BK.W_GATE[0], BK.LIDAR_CONST[0],
                                                   BK.REFLECT_THRES)
            else:
                c.map_set_points(BK.f4(W["surf_map"]))
                v, pl, sc = c.correspond_surf(BK.f4(W["surf_q"])[:n], W["pose"], 1.0, BK.SURF_DIST_THRES, BK.W_GATE[1], BK.LIDAR_CONST[1])
            return {"v": b(v), "pl": b(pl), "sc": b(sc), "blk": b(c.backend_surf_block(body, cauchy_b=1.0))}
        return f
    for kind, kinds in (("edge", ("48", "32")), ("surf", ("48", "32")), ("refl", ("48",))):
        inputs = {"large": corr_run(kind, ALL), "small": corr_run(kind, 40), "n1": corr_run(kind, 1), "n129": corr_run(kind, 129)}
        ops.append(Op(f"correspond_{kind}", kinds, inputs, nxt_s2m))
    return ops


@functools.lru_cache(None)
def catalogue():
    return [*_ops_decode(), *_ops_extract(), *_ops_vg(), *_ops_s2m(), *_ops_map(), *_ops_backend()]


def ops_of(kind):
    return [op for op in catalogue() if kind in op.kinds]


def by_name(name):
    return next(op for op in catalogue() if op.name == name)
