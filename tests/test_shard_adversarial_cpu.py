"""CPU tier of the sharded map: on every adversarial partition (tests/shard_adversarial.py), the 5-NN of each owned query on the
rank's shard (sharding.shard_mask, halo = the search radius) equals its 5-NN on the whole map, both by the plain gated reference
(knn_reference.reference_knn5: distance bits and map order) and by the oracle's find_surf_corr (accept flags, planes, neighbours).
The worlds are also checked for the tight situations they are built for, so a silently benign world fails here."""
import numpy as np
import pytest

import shard_adversarial as S
from knn_reference import reference_knn5
from liliom_b200 import sharding

WORLDS = S.worlds()
NEAR = 2.0 ** -21                          # a few fp32 steps from 1.0 (the spacing is 2^-24 below 1.0, 2^-23 above)
IDENT = np.array([1.0, 0, 0, 0, 0, 0, 0])


def _cube(xyz, block):
    xyz = np.asarray(xyz, np.float32)
    inv = np.float32(1.0 / block)
    return np.stack([np.floor(xyz[..., 0] * inv), np.floor(xyz[..., 1] * inv), np.floor(xyz[..., 2] * inv + np.float32(0.5))], -1)


@pytest.mark.parametrize("name,block,base", WORLDS, ids=[w[0] for w in WORLDS])
def test_shard_knn_equals_whole_map(oracle, name, block, base):
    w = S.world(block, base)
    m, q = w["map"], w["queries"]
    idx_all, sqd_all, _ = reference_knn5(q, m, S.TAU0)
    tree = oracle.KdTree(m)
    cnt_all, v_all, pl_all, oi_all, _ = oracle.find_surf_corr(tree, q, IDENT)
    accepted = idx_all[:, 4] >= 0
    # the situations the world is built for
    k, d5 = w["kind"], w["d5"]
    across_ok = np.array([a >= 0 and (_cube(m[a, :3], block) != _cube(q[i, :3], block)).any() for i, a in enumerate(w["across"])])
    in_5th = np.array([accepted[i] and w["across"][i] in idx_all[i] for i in range(len(q))])
    tight_in = int(((k == "in") & (d5 >= 1.0 - NEAR) & across_ok & in_5th & accepted).sum())
    tight_out = int(((k == "out") & (d5 <= 1.0 + NEAR) & across_ok & ~accepted).sum())
    ties = int(((k == "tie") & across_ok & accepted).sum())
    exact = int(((k == "in") & (d5 == S.TAU0)).sum() + ((k == "out") & (d5 == 1.0)).sum())
    print(f"{name}: {len(m)} map points, {len(q)} queries ({int(accepted.sum())} accepted); neighbour across a face within "
          f"{NEAR:.1e} of the gate: {tight_in} accepted, {tight_out} rejected ({exact} exactly one step); {ties} ties across a face")
    assert tight_in >= 4 and tight_out >= 3 and ties >= 6
    assert ((k == "corner") & accepted).sum() >= 20
    # eight cubes around the corner queries (at x = y = 0 a denormal times 1/block rounds to -0: one ulp below 0 is in cube 0)
    assert len(np.unique(_cube(q[k == "corner", :3], block), axis=0)) == (2 if base == (0.0, 0.0) else 8)
    for nranks in S.RANKS:
        own = sharding.owner_of(q[:, :3], nranks, block)
        for r in range(nranks):
            keep = sharding.shard_mask(m[:, :3], nranks, r, halo=S.GATE_HALO, block=block)
            gl = np.flatnonzero(keep)
            mine = own == r
            if not mine.any():
                continue
            idx, sqd, _ = reference_knn5(q[mine], m[keep], S.TAU0)
            idx = np.where(idx >= 0, gl[np.maximum(idx, 0)], -1)
            assert np.array_equal(idx, idx_all[mine]), f"{name} n={nranks} rank {r}: 5-NN on the shard"
            assert np.array_equal(sqd.view(np.uint32), sqd_all[mine].view(np.uint32)), f"{name} n={nranks} rank {r}: distances"
            cnt, v, pl, oi, _ = oracle.find_surf_corr(oracle.KdTree(m[keep]), q[mine], IDENT)
            assert np.array_equal(v, v_all[mine]), f"{name} n={nranks} rank {r}: oracle accept flags"
            assert np.array_equal(pl.view(np.uint32)[v == 1], pl_all[mine].view(np.uint32)[v == 1]), f"{name}: oracle planes"
            ok = v == 1
            assert np.array_equal(gl[oi[ok]], oi_all[mine][ok]), f"{name} n={nranks} rank {r}: oracle neighbours"


@pytest.mark.parametrize("block", S.BLOCKS)
def test_halo_frames_straddle_the_push_halo(block):
    """the frames of the map-maintenance check put points on both sides of the push halo of some rank, at every base"""
    for bx, by in S.BASES:
        f = S.halo_frame(block, (bx, by))
        for nranks in S.RANKS:
            wide = [sharding.shard_mask(f, nranks, r, halo=float(S.PUSH_HALO), block=block) for r in range(nranks)]
            assert any(0 < k.sum() < len(f) for k in wide), (block, bx, by, nranks)
