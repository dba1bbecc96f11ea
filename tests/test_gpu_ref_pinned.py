"""The device against the reference's own code directly, not through the oracle.  The reference's front-end and odometry
translation units, compiled against oracle/ref/'s shims, published the clouds whose digests tests/golden/ref_pinned.json holds
(tests/ref_cases.py: the cases, their inputs and the fixture format; test_ref_pinned_cpu.py checks the file against the compiled
reference wherever it is built).  Here every case's inputs are rebuilt, their digest checked against the fixture's, the device
run on them with the q the reference published with, and every cloud it returns must have the reference's digest: bit for bit,
a NaN equal to any NaN.  Nothing here needs the reference tree or oracle/_ref/."""
import numpy as np
import pytest

import ref_cases as RC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return RC.load_golden()


def _q(golden, case):
    return RC.q_of(golden[case.id]["q"])


def _expect(golden, case, **got):
    want = golden[case.id]
    assert RC.digest(case.inputs) == want["in"], f"{case.id}: the inputs differ from those the fixture was written from"
    for k, v in got.items():
        assert RC.digest(v) == want[k], (case.id, k, f"{len(v)} points, the reference published {want[k][0]}")


def _rot_ctx(line_num, ds_rate):
    import liliom_b200 as L
    p = L.default_params(1)
    p.line_num, p.ds_rate = line_num, ds_rate
    return L.Context(p)


def test_extract_horizon_against_reference_node(ctx48, world_small, golden):
    """extract_horizon against the Horizon node's published clouds on world_small and every hz_adversarial sweep"""
    cases = RC.hz_cases(world_small)
    for c in cases:
        s, e, cut = ctx48.extract_horizon(c.pts, _q(golden, c))
        _expect(golden, c, surf=s, edge=e, cut=cut)
    print(f"extract_horizon: {len(cases)} sweeps bit for bit against the reference node")


def test_extract_horizon_livox_against_reference_chain(ctx48, golden):
    """convert_livox against FormatConvert, and extract_horizon_livox against FormatConvert's cloud through the Horizon node"""
    cases = RC.livox_cases()
    for c in cases:
        stride = c.stride if c.stride != 20 else None
        conv = ctx48.convert_livox(c.recs, stride)
        s, e, cut = ctx48.extract_horizon_livox(c.recs, _q(golden, c), stride)
        _expect(golden, c, conv=conv, surf=s, edge=e, cut=cut)
    print(f"Livox chain: {len(cases)} messages bit for bit against FormatConvert + the Horizon node")


def test_extract_rot_against_reference_node(world_small, golden):
    """extract_rot and extract_rot_pc2 against the ROT node (typed cloud and the driver's PointCloud2) at 16 / 32 / 64 lines,
    ds_rate 1 and 2, both q_lb"""
    cases = RC.rot_world_cases(world_small)
    ctxs = {}
    try:
        for c in cases:
            ctx = ctxs.get((c.ln, c.ds)) or ctxs.setdefault((c.ln, c.ds), _rot_ctx(c.ln, c.ds))
            q = _q(golden, c)
            s, e, cut = ctx.extract_rot_pc2(RC.velodyne_msg(c.pts), q, c.qlb) if c.pc2 else ctx.extract_rot(c.pts, q, c.qlb)
            _expect(golden, c, surf=s, edge=e, cut=cut)
    finally:
        for ctx in ctxs.values():
            ctx.close()
    print(f"extract_rot: {len(cases)} sweeps bit for bit against the reference node")


def test_extract_rot_adversarial_against_reference_node(oracle, golden):
    """every rot_adversarial sweep: the ring-ordered cloud bit for bit, the features where no sort range holds tied candidates
    (the reference's std::sort orders those its own way)"""
    cases = RC.rot_adv_cases()
    n_feat = 0
    for c in cases:
        sw = c.sw
        q = _q(golden, c)
        ctx = _rot_ctx(sw["line_num"], sw["ds_rate"])
        try:
            s, e, cut = ctx.extract_rot(c.pts, q, sw["q_lb"])
        finally:
            ctx.close()
        _, _, _, cut_o, _, curv = oracle.extract_rot(c.pts, q, sw["q_lb"], sw["line_num"], sw["ds_rate"])
        if RC.rot_tied(cut_o, curv, sw["line_num"]):
            _expect(golden, c, cut=cut)
        else:
            _expect(golden, c, cut=cut, surf=s, edge=e); n_feat += 1
    assert len(cases) >= 30 and n_feat >= 2
    print(f"extract_rot: {len(cases)} adversarial sweeps, every ring-ordered cloud and {n_feat} sweeps' features bit for bit")


@pytest.mark.parametrize("variant", [0, 1])
def test_undistort_against_reference(ctx48, ctx32, golden, variant):
    """undistort against LidarOdometry::undistortion on the intensity and quaternion edges"""
    ctx = ctx48 if variant == 0 else ctx32
    for c in RC.undist_cases(variant):
        _expect(golden, c, out=ctx.undistort(c.pts, c.trans, c.q))


@pytest.mark.parametrize("variant", [0, 1])
def test_find_surf_corr_against_reference(world_small, golden, variant):
    """find_surf_corr against findCorrespondingSurfFeatures: the accepted points in order and their planes"""
    import liliom_b200 as L
    for c in RC.surf_cases(variant, world_small):
        ctx = L.Context(variant=variant)
        try:
            ctx.map_set_points(c.m4)
            valid, plane, _, _, _ = ctx.find_surf_corr(c.feats, c.pose)
        finally:
            ctx.close()
        v = valid.astype(bool)
        _expect(golden, c, pts=c.feats[v], plane=np.ascontiguousarray(plane[v], np.float32))


@pytest.mark.parametrize("variant", [0, 1])
def test_map_update_against_build_local_map(oracle, world_small, golden, variant):
    """map_update over 26 scans against buildLocalMap + downSampleCloud: after the frames of scans 1 .. k-1 the device's map is
    the map the reference matched scan k against"""
    import liliom_b200 as L
    c = RC.map_case(variant, world_small)
    ctx = L.Context(variant=variant)
    try:
        for k, (s, pose) in enumerate(c.steps):
            if k >= 2:
                _expect(golden, c, **{f"map{k}": ctx.map_download_cloud()})
            if k >= 1:
                ds = oracle.voxelgrid(s, 0.4) if len(s) else s
                _expect(golden, c, **{f"ds{k}": ds})
                ctx.map_update(ds, pose)
    finally:
        ctx.close()


@pytest.mark.parametrize("variant", [0, 1])
def test_preprocessing_node_against_reference_node(world_small, golden, variant):
    """liliom_pre_* (the host mirror of the Preprocessing node) against the compiled node over one IMU + cloud sequence: the
    published clouds and q_iMU bit for bit (processIMU, the wait gates and the queue included)"""
    import liliom_b200 as L
    for c in RC.node_cases(variant, world_small):
        ctx = L.Context(variant=variant)
        node = L.PreprocessingNode(ctx)
        try:
            for st, gy in c.stream:
                node.imu(st, gy)
            res = [node.cloud(stamp, cl) for stamp, cl in c.seq]
            assert res[0] is None and res[1] is None and res[2] is not None, c.id
            _, s, e, cut, q = res[2]
            assert RC.q_hex(q) == golden[c.id]["q"], (c.id, q)
            _expect(golden, c, surf=s, edge=e, cut=cut)
        finally:
            node.close(); ctx.close()
