"""GPU tier for two rules every entry point of the C ABI shares.

The caller-buffer contract of the download entry points: *n_out is the size; out == NULL is a size query that returns OK; a
capacity one short of the size returns LILIOM_E_CAPACITY with the size reported and leaves the caller's buffer byte for byte
untouched; a capacity equal to the size returns the same bytes as a download into a larger buffer.  Checked in both point
layouts for liliom_map_download, liliom_map_download_cloud, liliom_bmap_download (both layers), liliom_kf_cloud,
liliom_global_map (filtered and declined), the surf_last_ds output of liliom_odometry and liliom_backend_window_corr (both kinds).

The context's lifetime: a context that ran every subsystem gives all of its device memory back when it is destroyed."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
N_KF = 8
TINY_LEAF = 1e-4          # PCL declines every keyframe-sized cloud at this leaf: the global map is the transformed input


def _vp(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


@pytest.fixture(scope="module")
def stores():
    """per point layout: a context with an odometry map (map_update of the keyframes' surf clouds), the keyframe store with full
    clouds, the local map and a resident window"""
    import liliom_b200 as L
    from liliom_b200 import synth
    out = {}
    for stride, variant in ((48, 0), (32, 1)):
        seq = synth.make_keyframe_sequence(N_KF, stride=stride, full=True)
        bp = L.backend_default_params(variant)
        c = L.Context(variant=variant)
        poses = [p for _, _, p, _ in seq]
        for i, (e, s, p, f) in enumerate(seq):
            c.map_update(s, p)
            assert c.kf_add(bp, e, s, download=False)[0] == i
            c.kf_add_full(bp, i, f)
        c.bmap_build(bp, list(range(N_KF)), poses)
        c.backend_window_correspond(bp, [5, 6, 7], poses[5:])
        out[stride] = (c, seq, poses)
    yield out
    for c, _, _ in out.values():
        c.close()


def _raw(sizes):
    """A call through the C ABI: run(c, seq, poses, cap, alloc) -> (rc, reported size, bytes of the output buffers or None).
    alloc = None passes NULL outputs; otherwise every output gets max(alloc, 1) sentinel-filled elements."""
    def deco(fn):
        def run(c, seq, poses, cap, alloc):
            bufs = None if alloc is None else [np.full(max(alloc, 1) * s(c), SENTINEL, np.uint8) for s in sizes]
            n = C.c_int(-7)
            rc = fn(c, seq, poses, cap, bufs, n)
            return rc, n.value, None if bufs is None else b"".join(b.tobytes() for b in bufs)
        run.sizes = sizes
        return run
    return deco


def _lib():
    import liliom_b200 as L
    return L._binding.lib()


STRIDE = lambda c: c.stride      # noqa: E731


def _one(bufs):
    return None if bufs is None else _vp(bufs[0])


@_raw([lambda c: 16])
def _map_download(c, seq, poses, cap, bufs, n):
    return _lib().liliom_map_download(c._h, _one(bufs), cap, C.byref(n))


@_raw([STRIDE])
def _map_download_cloud(c, seq, poses, cap, bufs, n):
    return _lib().liliom_map_download_cloud(c._h, _one(bufs), cap, C.byref(n))


def _bmap_download(layer):
    @_raw([STRIDE])
    def run(c, seq, poses, cap, bufs, n):
        return _lib().liliom_bmap_download(c._h, layer, _one(bufs), cap, C.byref(n))
    return run


@_raw([STRIDE])
def _kf_cloud(c, seq, poses, cap, bufs, n):
    ids = np.array([1, 2, 3], np.int32)
    p = np.ascontiguousarray(np.array(poses)[ids])
    return _lib().liliom_kf_cloud(c._h, _ip(ids), _dp(p), len(ids), 0.4, _one(bufs), cap, C.byref(n))


def _global_map(leaf):
    @_raw([STRIDE])
    def run(c, seq, poses, cap, bufs, n):
        import liliom_b200 as L
        ids = np.array([0, 2, 4], np.int32)
        p = np.ascontiguousarray(np.array(poses)[ids])
        return _lib().liliom_global_map(c._h, L.KF_FULL, _ip(ids), _dp(p), len(ids), None, leaf, _one(bufs), cap, C.byref(n))
    return run


@_raw([STRIDE])
def _odometry_ds(c, seq, poses, cap, bufs, n):
    import liliom_b200 as L
    surf = np.ascontiguousarray(seq[3][1])
    pose = np.array(poses[3], np.float64)
    return _lib().liliom_odometry(c._h, _vp(surf), len(surf), _dp(pose), 1, 4, L.MODE_GN, None, _one(bufs), cap, C.byref(n))


def _window_corr(kind):
    sizes = [lambda c: 1, lambda c: 12, lambda c: 12] if kind == 0 else [lambda c: 1, lambda c: 16, lambda c: 8]

    @_raw(sizes)
    def run(c, seq, poses, cap, bufs, n):
        v, a, b = (None, None, None) if bufs is None else (_vp(x) for x in bufs)
        return _lib().liliom_backend_window_corr(c._h, 1, kind, v, a, b, cap, C.byref(n))
    return run


CASES = {
    "map_download": _map_download,
    "map_download_cloud": _map_download_cloud,
    "bmap_download_edge": _bmap_download(0),
    "bmap_download_surf": _bmap_download(1),
    "kf_cloud": _kf_cloud,
    "global_map": _global_map(0.3),
    "global_map_declined": _global_map(TINY_LEAF),
    "odometry_ds": _odometry_ds,
    "window_corr_edge": _window_corr(0),
    "window_corr_surf": _window_corr(1),
}


@pytest.mark.parametrize("stride", [48, 32])
@pytest.mark.parametrize("case", list(CASES))
def test_caller_buffer_contract(stores, stride, case):
    import liliom_b200 as L
    c, seq, poses = stores[stride]
    run = CASES[case]
    rc, m, _ = run(c, seq, poses, 0, None)                          # size query
    assert rc == L._binding.OK and m > 1, (rc, m)
    rc, n, big = run(c, seq, poses, m + 8, m + 8)                  # into a larger buffer
    assert (rc, n) == (L._binding.OK, m)
    rc, n, short = run(c, seq, poses, m - 1, m)                    # one short: E_CAPACITY, the size, nothing written
    assert (rc, n) == (L._binding.E_CAPACITY, m)
    assert short == bytes([SENTINEL]) * len(short)
    rc, n, exact = run(c, seq, poses, m, m)                        # exact: the same bytes as the larger download
    assert (rc, n) == (L._binding.OK, m)
    off_b = off_e = 0
    for s in run.sizes:
        w = s(c)
        assert exact[off_e:off_e + m * w] == big[off_b:off_b + m * w]
        assert big[off_b + m * w:off_b + (m + 8) * w] == bytes([SENTINEL]) * (8 * w)     # nothing past the size
        off_b += (m + 8) * w
        off_e += m * w


# ---------------------------------------------------------------- lifetime
def _cycle(world, seq):
    """one context through every subsystem, then destroyed"""
    import liliom_b200 as L
    bp = L.backend_default_params(0)
    c = L.Context(variant=0)
    surf, _, _ = c.extract_horizon(world["hz"], world["q_hz"])
    poses = [p for _, _, p, _ in seq]
    for e, s, p, f in seq:
        c.map_update(s, p)
        kid, _, _ = c.kf_add(bp, e, s, download=False)
        c.kf_add_full(bp, kid, f)
    c.odometry(surf, poses[0], 2, 4, mode=L.MODE_GN)
    ids = list(range(len(seq)))
    c.bmap_build(bp, ids, poses)
    c.backend_window_correspond(bp, ids[-3:], poses[-3:])
    c.backend_window_blocks(poses[-3:])
    c.backend_window_corr(0, 1)
    assert len(c.global_map(L.KF_FULL, ids, poses, 0.3)) > 0
    c.loop_align([ids[-1]], [poses[-1]], ids[:-1], poses[:-1], 0.4)
    src, tgt = c.kf_cloud([ids[-1]], [poses[-1]], 0.4), c.kf_cloud(ids[:-1], poses[:-1], 0.4)
    c.icp_align(src, tgt)
    c.close()


def test_destroy_gives_back_all_device_memory(world_small):
    import torch
    from liliom_b200 import synth
    seq = synth.make_keyframe_sequence(N_KF, stride=48, full=True)
    _cycle(world_small, seq)                                        # warm-up: loads the library's modules
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    _cycle(world_small, seq)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 <= (2 << 20), (free0, free1)
