"""Mesh metrics without a GPU: the oracle's sampler and ground-truth mesh, read_ply against write_ply and malformed
files, reconstruct.py's --gt_mesh refusals, and the kernels' register report."""
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import mesh_oracle as MO
from oracle import volume_oracle as VO

ROOT = Path(__file__).resolve().parents[1]
CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)


def test_oracle_samples_lie_on_their_triangles_and_counts_match_the_area():
    rng = np.random.default_rng(0)
    v = rng.uniform(-1, 1, (40, 3)).astype(np.float32)
    f = rng.integers(0, 40, (60, 3))
    n, p = MO.sample_surface(v, f, 500.0, 3, 1)
    t = np.repeat(np.arange(len(f)), n)
    a, b, c = (v[f[t, q]].astype(np.float64) for q in range(3))
    # barycentric coordinates by least squares: non-negative, summing to 1, and the residual at fp32 rounding
    M = np.stack([b - a, c - a], -1)
    uv = np.linalg.lstsq(M[0], (p[0] - a[0]), rcond=None)[0] if len(p) == 1 else \
        np.stack([np.linalg.lstsq(M[i], p[i] - a[i], rcond=None)[0] for i in range(len(p))])
    res = np.abs(a + np.einsum("ijk,ik->ij", M, uv) - p).max(1)
    assert np.all(res <= 1e-6) and np.all(uv >= -1e-5) and np.all(uv.sum(1) <= 1 + 1e-5)
    # E[n_t] = A_t rho exactly: over 400 seeds the mean total lies within 4 standard errors of sum(A) rho
    area = MO.face_areas(v, f)
    totals = np.array([MO.sample_counts(v, f, 37.0, s).sum() for s in range(400)])
    assert abs(totals.mean() - 37.0 * area.sum()) <= 4 * totals.std(ddof=1) / np.sqrt(len(totals))


def test_generator_is_splitmix64():
    # splitmix64's published first outputs from state 0 (x += golden gamma, then the finaliser)
    assert int(MO.splitmix64(np.array([0], np.uint64))[0]) == 0xE220A8397B1DCDAF
    assert 0.0 <= MO.draw(MO.stream_key(0, 0), np.arange(1000, dtype=np.uint64), 5).min()
    assert MO.draw(MO.stream_key(0, 0), np.arange(1000, dtype=np.uint64), 5).max() < 1.0


def test_sphere_room_mesh_is_closed_and_exact():
    v, f = MO.sphere_room_mesh(CENTER, RADIUS, ROOM_LO, ROOM_HI, 4)
    _, mult = VO.mesh_edges(f)
    assert np.all(mult == 2)
    r = np.abs(np.linalg.norm(v - np.asarray(CENTER), axis=1) - RADIUS)
    on_room = np.min(np.abs(np.concatenate([v - np.asarray(ROOM_LO), v - np.asarray(ROOM_HI)], 1)), 1)
    inside = np.all((v >= np.asarray(ROOM_LO) - 1e-12) & (v <= np.asarray(ROOM_HI) + 1e-12), 1)
    assert np.all(np.minimum(r, on_room) <= 1e-12) and inside.all()
    # the room wound inward, the sphere outward: signed volume = sphere - room
    want = 4 / 3 * np.pi * RADIUS ** 3 - 27.0
    assert abs(VO.signed_volume(v, f) - want) < 0.02


def _ply(tmp_path, header, body: bytes, name="m.ply"):
    p = tmp_path / name
    p.write_bytes(("\n".join(["ply"] + header + ["end_header"]) + "\n").encode() + body)
    return p


@pytest.mark.parametrize("color", [False, True])
def test_read_ply_round_trips_write_ply(tmp_path, color):
    from omnidata_b200.volume import read_ply, write_ply
    rng = np.random.default_rng(1)
    v = rng.standard_normal((70, 3)).astype(np.float32)
    f = rng.integers(0, 70, (90, 3)).astype(np.int32)
    c = rng.random((70, 3)) if color else None
    write_ply(tmp_path / "a.ply", v, f, c)
    V, F, C = read_ply(tmp_path / "a.ply")
    assert np.array_equal(V, v) and np.array_equal(F, f) and V.dtype == np.float32 and F.dtype == np.int32
    assert (C is None) == (not color)
    if color:
        assert np.array_equal(np.rint(C * 255.0).astype(np.uint8), np.rint(np.clip(c, 0, 1) * 255).astype(np.uint8))
    write_ply(tmp_path / "b.ply", V, F, C)
    assert (tmp_path / "a.ply").read_bytes() == (tmp_path / "b.ply").read_bytes()
    V0, F0, _ = read_ply(_ply(tmp_path, ["format binary_little_endian 1.0", "element vertex 0", "property float x",
                                         "property float y", "property float z", "element face 0",
                                         "property list uchar int vertex_indices"], b""))
    assert V0.shape == (0, 3) and F0.shape == (0, 3)


def test_read_ply_ascii_double_quads_and_extra_properties(tmp_path):
    from omnidata_b200.volume import read_ply
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0.5, 0.5, 1.0]], np.float64)
    header = ["format ascii 1.0", "comment made by hand", "element vertex 5", "property double x", "property double y",
              "property double z", "property float nx", "property uchar red", "property uchar green",
              "property uchar blue", "property ushort label", "element face 2",
              "property list uchar uint vertex_indices", "element edge 1", "property int vertex1",
              "property int vertex2"]
    lines = [f"{x} {y} {z} 0.5 {10 * i} 20 30 7" for i, (x, y, z) in enumerate(v)]
    lines += ["4 0 1 2 3", "3 0 1 4", "0 1"]
    V, F, C = read_ply(_ply(tmp_path, header, ("\n".join(lines) + "\n").encode()))
    assert np.array_equal(V, v.astype(np.float32))
    assert F.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 4]]
    assert np.allclose(C[:, 0] * 255, [0, 10, 20, 30, 40])
    # binary: double coordinates, an extra int property, quads with an int count
    rec = np.zeros(5, [("x", "<f8"), ("q", "<i4"), ("y", "<f8"), ("z", "<f8")])
    rec["x"], rec["y"], rec["z"] = v.T
    quads = np.array([(4, (0, 1, 2, 3)), (4, (1, 2, 3, 4))], [("n", "<i4"), ("i", "<i4", (4,))])
    header = ["format binary_little_endian 1.0", "element vertex 5", "property double x", "property int q",
              "property double y", "property double z", "element face 2", "property list int int vertex_indices"]
    V, F, C = read_ply(_ply(tmp_path, header, rec.tobytes() + quads.tobytes()))
    assert np.array_equal(V, v.astype(np.float32)) and C is None
    assert F.tolist() == [[0, 1, 2], [0, 2, 3], [1, 2, 3], [1, 3, 4]]
    # mixed polygon sizes
    mixed = np.array([3, 0, 1, 2], "<u1").tobytes()[:1] + np.array([0, 1, 2], "<i4").tobytes() + \
        np.array([4], "<u1").tobytes() + np.array([0, 1, 2, 3], "<i4").tobytes()
    header[-1] = "property list uchar int vertex_indices"
    V, F, _ = read_ply(_ply(tmp_path, header, rec.tobytes() + mixed))
    assert F.tolist() == [[0, 1, 2], [0, 1, 2], [0, 2, 3]]
    # triangles and quads whose index bytes equal 3, the triangles' count: read at the triangles' stride, the first
    # quad's count is still read at its own offset, so the fast path is refused and nothing misaligned is accepted
    polys = [(3, 3, 3)] * 3 + [(3, 3, 3, 3)] * 2 + [(0, 1, 2)]
    blob = b"".join(np.array([len(p)], "<u1").tobytes() + np.array(p, "<i4").tobytes() for p in polys)
    header[-2] = "element face 6"
    V, F, _ = read_ply(_ply(tmp_path, header, rec.tobytes() + blob))
    assert F.tolist() == [[3, 3, 3]] * 7 + [[0, 1, 2]]


def test_read_ply_refusals(tmp_path):
    from omnidata_b200.volume import read_ply, write_ply
    rng = np.random.default_rng(2)
    write_ply(tmp_path / "ok.ply", rng.random((10, 3)), rng.integers(0, 10, (5, 3)))
    data = (tmp_path / "ok.ply").read_bytes()
    cases = {
        "big-endian": data.replace(b"binary_little_endian", b"binary_big_endian"),
        "x, y, z": data.replace(b"property float z", b"property float w"),
        "truncated": data[:-7],
        "outside": data[:-4] + np.array([10], "<i4").tobytes(),
        "not a PLY": b"solid cube\n",
        "malformed": data.replace(b"element vertex 10", b"element vertex ten"),
        "negative": data.replace(b"element face 5", b"element face -5"),
    }
    for what, blob in cases.items():
        p = tmp_path / "bad.ply"
        p.write_bytes(blob)
        with pytest.raises(ValueError, match=re.escape(str(p))) as e:
            read_ply(p)
        assert what in str(e.value), (what, str(e.value))


BASE = ["--img_path", "imgs", "--intrinsics", "500,500,320,240", "--voxel", "0.02", "--out", "m.ply",
        "--synthetic_weights", "--sparse_path", "sp"]


def test_reconstruct_gt_mesh_arguments():
    import reconstruct
    a = reconstruct.parse_args(BASE + ["--pose_path", "p", "--gt_mesh", "gt.ply", "--gt_cull",
                                       "--eval_thresholds", "0.02,0.05", "--eval_density", "2e4"])
    assert a.gt_mesh == "gt.ply" and a.gt_cull and a.eval_thresholds == (0.02, 0.05) and a.eval_density == 2e4
    assert reconstruct.parse_args(BASE).gt_mesh is None
    for bad in (["--gt_mesh", "gt.ply"],                                   # no --pose_path: frame 0's world
                ["--pose_path", "p", "--gt_cull"],                          # --gt_cull without --gt_mesh
                ["--pose_path", "p", "--gt_mesh", "g", "--eval_thresholds", "0.1,0.2,0.3,0.4,0.5"],
                ["--pose_path", "p", "--gt_mesh", "g", "--eval_thresholds", "-0.1"],
                ["--pose_path", "p", "--gt_mesh", "g", "--eval_density", "0"]):
        with pytest.raises(SystemExit):
            reconstruct.parse_args(BASE + bad)


def test_mesh_metrics_kernels_have_no_stack_frames_or_spills(tmp_path):
    from omnidata_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "mesh_metrics.cu"), "-o",
           str(tmp_path / "mesh_metrics.o")]
    try:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    except FileNotFoundError:
        pytest.skip("nvcc not found")
    assert r.returncode == 0, r.stdout
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    assert len(frames) >= 20
    assert all(f == ("0", "0", "0") for f in frames), r.stdout
