"""The single-launch scan VoxelGrid (k_vg_coop) against the sort chain, byte for byte, at the edges of its schedule: a voxel
with exactly as many members as a warp orders in shared memory and one more, voxel counts around one voxel round of the grid
(one warp per voxel) and around the key list a block ranks from shared memory, PCL's overflow box, and back-to-back calls of
different sizes (hash slots handed back between launches).  The sort chain is the same library's multi-launch filter, taken
by padding the cloud with NaN points beyond the cooperative filter's size limit (non-finite points are dropped by both)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# voxelgrid.cu
VGC_NCAP = 32768      # larger clouds take the sort chain
VGC_VCAP = 256        # members per voxel the cooperative filter orders in shared memory; one more: it declines
VGC_UKEYS = 8192      # voxel keys a block ranks from shared memory; more: read through L2
VGC_WARPS = 16        # warps per block (one block per SM); one voxel round = SMs x VGC_WARPS voxels
LEAF = 0.4


@pytest.fixture(scope="module")
def ctxs():
    import liliom_b200 as L
    a, b, c, d = L.Context(variant=0), L.Context(variant=0), L.Context(variant=1), L.Context(variant=1)
    yield {48: (a, b), 32: (c, d)}      # (filter under test, sort-chain reference) per point stride
    for x in (a, b, c, d):
        x.close()


@pytest.fixture(scope="module")
def voxel_round():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * VGC_WARPS


def _cloud(dtype, n_vox, seed, heavy=0, span=64):
    """n_vox distinct occupied voxels (1-3 members each; voxel 0 gets `heavy` members when heavy > 0), shuffled,
    every point well inside its cell, random payload fields."""
    rng = np.random.default_rng(seed)
    flat = rng.choice(span ** 3, n_vox, replace=False)
    cells = np.stack([flat % span, (flat // span) % span, flat // (span * span)], 1) - span // 2
    members = rng.integers(1, 4, n_vox)
    if heavy:
        members[0] = heavy
    idx = np.repeat(np.arange(n_vox), members)
    rng.shuffle(idx)
    xyz = (cells[idx] * LEAF + rng.uniform(0.1, 0.3, (len(idx), 3))).astype(np.float32)
    out = np.zeros(len(idx), dtype)
    out["x"], out["y"], out["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    out["w"] = 1.0
    for f in dtype.names:
        if f not in ("x", "y", "z", "w"):
            out[f] = rng.uniform(-1.0, 1.0, len(idx)).astype(np.float32)
    return out


def _sort_chain(ref, cloud):
    pad = np.zeros(VGC_NCAP + 1 - len(cloud), cloud.dtype)
    pad["x"] = np.nan
    return ref.voxelgrid(np.concatenate([cloud, pad]), LEAF)


def _run(c, cloud):
    """(output, cooperative): cooperative = the call was one launch (k_vg_coop), not the filter plus the sort chain."""
    c.counters(reset=True)
    out = c.voxelgrid(cloud, LEAF)
    return out, c.counters().launches == 1


def _check(ctxs, cloud, n_vox, coop):
    c, ref = ctxs[cloud.dtype.itemsize]
    out, was_coop = _run(c, cloud)
    exp = _sort_chain(ref, cloud)
    assert was_coop == coop
    assert len(out) == len(exp) == n_vox
    assert out.tobytes() == exp.tobytes()


@pytest.mark.parametrize("extra", [0, 1])
def test_voxel_with_vcap_members(ctxs, extra):
    import liliom_b200 as L
    cloud = _cloud(L.PT48, 300, seed=11 + extra, heavy=VGC_VCAP + extra)
    _check(ctxs, cloud, 300, coop=extra == 0)


@pytest.mark.parametrize("stride", [48, 32])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_voxel_count_around_one_round(ctxs, voxel_round, stride, delta):
    import liliom_b200 as L
    n_vox = voxel_round + delta
    _check(ctxs, _cloud(L.PT48 if stride == 48 else L.PT32, n_vox, seed=20 + delta), n_vox, coop=True)


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_voxel_count_around_shared_key_list(ctxs, delta):
    import liliom_b200 as L
    n_vox = VGC_UKEYS + delta
    _check(ctxs, _cloud(L.PT48, n_vox, seed=30 + delta), n_vox, coop=True)


def test_overflow_box_copies_input(ctxs, oracle):
    """PCL's index overflow (dx*dy*dz > INT_MAX): the filter declines and the output is the input, as PCL's."""
    import liliom_b200 as L
    cloud = _cloud(L.PT48, 500, seed=40, span=2048)
    c, _ = ctxs[48]
    out, was_coop = _run(c, cloud)
    assert not was_coop
    exp = oracle.voxelgrid(cloud, LEAF)
    assert len(out) == len(exp) == len(cloud)
    for f in ("x", "y", "z", "nx", "ny", "nz", "intensity", "curvature"):
        assert np.array_equal(out[f].view(np.uint32), exp[f].view(np.uint32)), f


@pytest.mark.parametrize("stride", [48, 32])
def test_back_to_back_sizes(ctxs, voxel_round, stride):
    """Consecutive calls of different sizes on one context (declined ones included): every call starts from a clean table."""
    import liliom_b200 as L
    dt = L.PT48 if stride == 48 else L.PT32
    c, ref = ctxs[stride]
    seq = [(voxel_round + 1, 0), (3, 0), (VGC_UKEYS + 1, 0), (200, VGC_VCAP + 1), (1, 0), (voxel_round - 1, VGC_VCAP),
           (2 * voxel_round + 5, 0), (40, 0)]
    clouds = [_cloud(dt, nv, seed=50 + k, heavy=h) for k, (nv, h) in enumerate(seq)]
    exps = [_sort_chain(ref, cl) for cl in clouds]
    for rep in range(2):
        for (nv, h), cl, exp in zip(seq, clouds, exps):
            out, was_coop = _run(c, cl)
            assert was_coop == (h <= VGC_VCAP)
            assert len(out) == nv and out.tobytes() == exp.tobytes()
