"""Sparse TSDF volume without a GPU: the oracle's block allocation on hand-built cases, the host's refusals,
reconstruct.py's argument parsing with and without --bounds, and the kernels' register report."""
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import sparse_volume_oracle as so

ROOT = Path(__file__).resolve().parents[1]
V = 0.125                      # 1 m blocks
K1 = (1.0, 1.0, 0.0, 0.0)      # a 1 x 1 image's pixel looks along +z


def _blocks(depth, K=K1, pose=np.eye(4), trunc=0.25, max_depth=10.0, origin=(0.0, 0.0, 0.0)):
    return {so.unpack_key(k) for k in so.frame_blocks(np.asarray(depth, np.float32), K, pose, origin, V, trunc,
                                                      max_depth)}


def test_pack_key_orders_by_z_then_y_then_x():
    b = [(0, 0, 1), (5, 0, 0), (0, 1, 0), (-3, -2, -1)]
    assert sorted(b, key=so.pack_key) == [(-3, -2, -1), (5, 0, 0), (0, 1, 0), (0, 0, 1)]
    for q in b + [(so.BLOCK_RANGE - 1, -so.BLOCK_RANGE + 1, 7)]:
        assert so.unpack_key(so.pack_key(q)) == q


def test_one_pixel_allocates_the_blocks_of_its_segment():
    # segment z in [2.5 - 0.25, 2.5 + 0.25] on the z axis: block z = 2 only; across the face z = 3 m: blocks 2 and 3
    assert _blocks([[2.5]]) == {(0, 0, 2)}
    assert _blocks([[2.9]]) == {(0, 0, 2), (0, 0, 3)}
    # negative side of the origin: floor, not truncation
    T = np.eye(4)
    T[:3, 3] = (-0.5, -0.5, -10.0)
    assert _blocks([[2.5]], pose=T) == {(-1, -1, -8)}


def test_segment_across_a_block_corner_allocates_the_eight_blocks():
    # the pixel at (1, 1) with fx = fy = 1, cx = cy = 0 looks along (1, 1, 1): points (z, z, z)
    K = (1.0, 1.0, 0.0, 0.0)
    depth = np.zeros((2, 2), np.float32)
    depth[1, 1] = 1.0
    got = _blocks(depth, K=K, trunc=0.25)
    assert got == {(x, y, z) for x in (0, 1) for y in (0, 1) for z in (0, 1)}


def test_max_depth_limits_allocation():
    assert _blocks([[4.0]], max_depth=4.0) == {(0, 0, 3), (0, 0, 4)}
    assert _blocks([[4.0]], max_depth=np.nextafter(4.0, 0.0)) == set()


@pytest.mark.parametrize("d", [np.nan, np.inf, 0.0, -1.0])
def test_bad_depth_allocates_nothing(d):
    assert _blocks([[d]]) == set()


def test_blocks_outside_the_range_are_never_allocated():
    T = np.eye(4)
    T[2, 3] = 8 * V * (so.BLOCK_RANGE - 1)
    assert _blocks([[0.5]], pose=T) == {(0, 0, so.BLOCK_RANGE - 1)}
    assert _blocks([[1.5]], pose=T) == set()            # the segment's far end is in block 2^20


def test_oracle_ids_follow_birth_then_key():
    vol = so.SparseVolume(V, trunc=0.25)
    d = np.array([[[2.5]], [[1.5]], [[2.5]]], np.float32)
    vol.allocate(d, K1, np.stack([np.eye(4)] * 3))
    assert [so.unpack_key(int(k)) for k in vol.keys] == [(0, 0, 2), (0, 0, 1)]
    assert vol.birth.tolist() == [0, 1]


def test_oracle_birth_mask_and_split_invariance():
    rng = np.random.default_rng(0)
    K = (20.0, 20.0, 7.5, 5.5)
    T = np.stack([np.eye(4)] * 4)
    for f in range(4):
        T[f, :3, 3] = (0.1 * f, 0.0, 0.0)
    d = (1.0 + 0.5 * rng.random((4, 12, 16))).astype(np.float32)
    d[1, :6] = 2.5                                                 # frame 1 reaches blocks frame 0 never saw
    one = so.SparseVolume(V, trunc=0.2)
    one.integrate(d, K, T)
    split = so.SparseVolume(V, trunc=0.2)
    for f in range(4):
        split.integrate(d[f:f + 1], K, T[f:f + 1])
    assert (one.keys == split.keys).all() and (one.birth == split.birth).all()
    assert np.array_equal(one.data, split.data)
    late = one.birth > 0
    assert late.any() and (one.data[late, 1] <= 3).all()            # born after frame 0: frame 0 never counts


def _volume_error(**kw):
    from omnidata_b200.volume import SparseTSDFVolume
    with pytest.raises(ValueError) as e:
        SparseTSDFVolume(device="cpu", **kw)
    return str(e.value)


def test_host_refusals():
    assert "block" in _volume_error(voxel=0.01, origin=(0.08 * so.BLOCK_RANGE, 0.0, 0.0))
    assert "voxel" in _volume_error(voxel=0.0)
    assert "trunc" in _volume_error(voxel=0.01, trunc=-1.0)
    assert "max_depth" in _volume_error(voxel=0.01, max_depth=float("inf"))
    assert "CUDA" in _volume_error(voxel=0.01)


def test_camera_centres_outside_the_block_range_are_refused():
    from omnidata_b200.volume import SparseTSDFVolume
    vol = SparseTSDFVolume.__new__(SparseTSDFVolume)
    vol.origin, vol.voxel, vol.trunc, vol.max_depth = (0.0, 0.0, 0.0), 0.01, 0.03, 10.0
    T = np.eye(4)
    vol._check_centres("t", T.reshape(1, 16))
    T[1, 3] = 0.08 * so.BLOCK_RANGE
    with pytest.raises(ValueError, match="block range"):
        vol._check_centres("t", T.reshape(1, 16))


BASE = ["--img_path", "imgs", "--intrinsics", "500,500,320,240", "--voxel", "0.02", "--out", "m.ply",
        "--synthetic_weights", "--sparse_path", "sp"]


def test_reconstruct_parses_without_bounds():
    import reconstruct
    a = reconstruct.parse_args(BASE)
    assert a.bounds is None and a.dims is None and a.origin == (0.0, 0.0, 0.0)


def test_reconstruct_parses_with_bounds_as_before():
    import reconstruct
    a = reconstruct.parse_args(BASE + ["--bounds=-1,-1,0,1,1,2"])
    assert a.origin == (-1.0, -1.0, 0.0) and a.dims == (101, 101, 101)
    with pytest.raises(SystemExit):
        reconstruct.parse_args(BASE + ["--bounds=1,1,1,0,2,2"])


def test_sparse_volume_kernels_have_no_stack_frames_or_spills(tmp_path):
    from omnidata_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "sparse_volume.cu"), "-o",
           str(tmp_path / "sparse_volume.o")]
    try:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    except FileNotFoundError:
        pytest.skip("nvcc not found")
    assert r.returncode == 0, r.stdout
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    assert len(frames) >= 14
    assert all(f == ("0", "0", "0") for f in frames), r.stdout
