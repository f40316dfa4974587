"""The photometric tracking term and the coloured raycast on the GPU (FrameTracker(photometric=...),
ops.track_frame, TSDFVolume.raycast(color=True), reconstruct.py --color --photometric; csrc/track.cu, csrc/volume.cu).

- Oracle parity on odd image sizes, affine on and off, with NaN, 0 and negative predictions, holes in the reference
  depth and NaN holes in its colour: one iteration gives the oracle's geometric and photometric term counts exactly
  and its pose and nodes within 1e-10; a full run agrees within 1e-7.
- The coloured raycast: depth identical to raycast, colour against the float64 oracle, NaN exactly where nothing is hit.
- The default path unchanged, determinism, CUDA-graph replay and the launch sequence of the photometric path.
- The textured single wall, the weakly constrained views of the chained path, and tracking against a fused colour
  model (frame to model, unposed and pose refinement), each against geometry alone in the same run.
- reconstruct.py --color --photometric without poses."""
import json

import numpy as np
import pytest
import torch

from oracle import color_volume_oracle as CO
from oracle import photometric_oracle as PO
from oracle import track_oracle as TO
from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
SIZE, F = (120, 160), 150.0
K = (F, F, (SIZE[1] - 1) / 2, (SIZE[0] - 1) / 2)
LAMBDA = 1e-2                               # the sweep's choice on this scene (DESIGN.md §6)
FINE = 0.0125


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _depth(pose, size=SIZE, k=K):
    return VO.sphere_room_depth(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI)


def _rgb(pose, size=SIZE, k=K):
    return CO.sphere_room_rgb(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32)


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(dev)


def _nodes(s, t):
    return torch.tensor([s, t], dtype=torch.float64, device=dev).reshape(1, 1, 1, 2)


def _aligner():
    import reconstruct
    from omnidata_b200.sparse import SparseDepthAligner
    return SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)


@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("hw", [(37, 53), (48, 64), (61, 83)])
def test_matches_the_oracle(hw, affine):
    from omnidata_b200.track import FrameTracker
    h, w = hw
    rng = np.random.default_rng(h * 7 + affine)
    k = (0.9 * w, 0.9 * w, (w - 1) / 2 + 0.3, (h - 1) / 2 - 0.2)
    ref = TO.camera_path(1, CENTER, seed=h)[0]
    truth = TO.perturb(ref, 0.02, np.radians(1.5), rng)
    d_ref = _depth(ref, hw, k).astype(np.float32)
    d_ref[rng.random(hw) < 0.03] = 0.0                                     # holes in the model
    c_ref = _rgb(ref, hw, k)
    c_ref[:, rng.random(hw) < 0.03] = np.nan                               # holes in its colour
    rgb = _rgb(truth, hw, k)
    s1, t1 = (rng.uniform(0.6, 1.8), rng.uniform(-0.2, 0.2)) if affine else (1.0, 0.0)
    pred = (s1 * _depth(truth, hw, k) + t1).astype(np.float32)
    bad = rng.random(hw)
    pred[bad < 0.02] = np.nan
    pred[(bad >= 0.02) & (bad < 0.03)] = 0.0
    pred[(bad >= 0.03) & (bad < 0.04)] = -1.0
    init = (1 / s1 * 1.01, -t1 / s1 + 0.01) if affine else None
    for iters in (1, 20):
        tr = FrameTracker(affine=affine, iterations=iters, photometric=LAMBDA)
        pose, nodes, rec = tr.track(_t(pred), _t(d_ref), k, ref, init_nodes=_nodes(*init) if affine else None,
                                    rgb=_t(rgb), ref_rgb=_t(c_ref))
        normals = tr._bufs["normals"][0].cpu().numpy()
        ig = tr._bufs["intensity"].cpu().numpy()
        want_ig = PO.intensity_gradient(d_ref, c_ref, normals)
        assert np.array_equal(ig, want_ig, equal_nan=True)               # (Y, g_u, g_v) bit for bit
        T, (s, t), orec = PO.track(pred, d_ref, k, ref, rgb, c_ref, None, init, affine=affine, iterations=iters,
                                   photometric=LAMBDA, normals=normals)
        rec = rec.cpu().numpy()
        tol = 1e-10 if iters == 1 else 1e-7
        print(f"{hw} affine={affine} iterations={iters}: {int(rec[0])} geometric and {int(rec[8])} photometric "
              f"terms (oracle {int(orec[0])}, {int(orec[8])}), status {int(rec[1])}, {int(rec[4])} run; pose diff "
              f"{np.abs(pose.cpu().numpy() - T).max():.2e}")
        assert rec.shape == (11,) and rec[1] == 0 and orec[1] == 0
        if iters == 1:
            assert rec[0] == orec[0] and rec[7] == orec[7] and rec[8] == orec[8]
        assert rec[4] == orec[4]
        assert np.abs(pose.cpu().numpy() - T).max() <= tol
        assert np.abs(nodes.reshape(2).cpu().numpy() - np.array([s, t])).max() <= tol
        assert abs(rec[2] - orec[2]) <= 1e-9 and abs(rec[3] - orec[3]) <= 1e-12
        assert abs(rec[9] - orec[9]) <= 1e-9 and abs(rec[10] - orec[10]) <= 1e-12


def _colour_volume(voxel, n_frames=20, size=SIZE, k=K):
    from omnidata_b200.volume import TSDFVolume
    T = VO.orbit_poses(n_frames, 1.2, CENTER)
    n = int(round(3.2 / voxel)) + 1
    vol = TSDFVolume((-1.6, -1.6, -1.6), voxel, (n, n, n), color=True, device=dev)
    vol.integrate(_t(np.stack([_depth(t, size, k) for t in T]).astype(np.float32)), k, T,
                  _t(np.stack([_rgb(t, size, k) for t in T])))
    return vol


def test_colour_raycast():
    vol = _colour_volume(0.05, 8, (48, 64), (60.0, 60.0, 31.5, 23.5))
    F, W, C = (x.cpu().numpy() for x in (vol.tsdf, vol.weight, vol.color))
    k = (70.0, 72.0, 40.3, 29.6)
    for seed, step in ((0, None), (1, 0.02)):
        pose = TO.camera_path(1, CENTER, seed=seed)[0]
        depth = vol.raycast(k, pose, (61, 83), step)
        got_d, got_c = vol.raycast(k, pose, (61, 83), step, color=True)
        again = vol.raycast(k, pose, (61, 83), step, color=True)
        assert torch.equal(got_d, depth)
        assert torch.equal(got_c.view(torch.int32), again[1].view(torch.int32))
        want_d, want_c = CO.raycast_color(F, W, C, vol.origin, vol.voxel, k, pose, (61, 83), step)
        assert np.array_equal(want_d, VO.raycast(F, W, vol.origin, vol.voxel, k, pose, (61, 83), step))
        got_c = got_c.cpu().numpy()
        hit = got_d.cpu().numpy() > 0
        assert hit.mean() > 0.5
        assert np.array_equal(np.isnan(got_c), np.broadcast_to(~hit, got_c.shape))
        assert np.array_equal(np.isnan(want_c), np.isnan(got_c))
        err = np.abs(got_c[:, hit] - want_c[:, hit]).max()
        print(f"coloured raycast, seed {seed}: {hit.sum()} hits, colour diff {err:.2e}")
        assert err <= 1e-6


def test_default_path_determinism_graph_and_launches():
    from omnidata_b200 import _capi
    from omnidata_b200.track import FrameTracker
    ref = TO.camera_path(1, CENTER)[0]
    truth = TO.perturb(ref, 0.03, np.radians(2.0), np.random.default_rng(4))
    pred, r = _t((1.3 * _depth(truth) - 0.1).astype(np.float32)), _t(_depth(ref).astype(np.float32))
    rgb, c_ref = _t(_rgb(truth)), _t(_rgb(ref))
    n0 = _nodes(0.78, 0.08)
    geo = [t.clone() for t in FrameTracker().track(pred, r, K, ref, init_nodes=n0)]
    zero = FrameTracker(photometric=0.0).track(pred, r, K, ref, init_nodes=n0)
    for x, y in zip(geo, zero):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))
    tr = FrameTracker(iterations=20, photometric=LAMBDA)
    out = [t.clone() for t in tr.track(pred, r, K, ref, init_nodes=n0, rgb=rgb, ref_rgb=c_ref)]
    assert out[2].shape == (11,) and int(out[2][1]) == 0 and out[2][8] > 0
    torch.cuda.synchronize()
    a0, l0 = torch.cuda.memory_stats(dev)["allocation.all.allocated"], _capi.launch_count()
    again = tr.track(pred, r, K, ref, init_nodes=n0, rgb=rgb, ref_rgb=c_ref)
    torch.cuda.synchronize()
    launches = _capi.launch_count() - l0
    assert torch.cuda.memory_stats(dev)["allocation.all.allocated"] == a0
    for x, y in zip(out, again):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))
    l1 = _capi.launch_count()
    FrameTracker(iterations=20).track(pred, r, K, ref, init_nodes=n0)
    assert launches == _capi.launch_count() - l1 + 1                    # one gradient kernel more
    print(f"launches per photometric FrameTracker.track: {launches}")
    for t in tr._bufs.values():
        if t.is_floating_point():
            t.fill_(float("nan"))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = tr.track(pred, r, K, ref, init_nodes=n0, rgb=rgb, ref_rgb=c_ref)
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(out, res):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))


def test_refusals_before_any_launch():
    from omnidata_b200 import _capi
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    d = torch.ones(24, 32, device=dev)
    c = torch.ones(3, 24, 32, device=dev)
    n0 = _nodes(1.0, 0.0)
    k = (30.0, 30.0, 15.5, 11.5)
    tr = FrameTracker(photometric=LAMBDA)
    vol = TSDFVolume((0, 0, 0), 0.1, (8, 8, 8), device=dev)
    n = _capi.launch_count()
    calls = [
        lambda: tr.track(d, d, k, np.eye(4), init_nodes=n0, rgb=c.double(), ref_rgb=c),     # dtype
        lambda: tr.track(d, d, k, np.eye(4), init_nodes=n0, rgb=c, ref_rgb=c.cpu()),        # device
        lambda: tr.track(d, d, k, np.eye(4), init_nodes=n0, rgb=c[:, :, :31], ref_rgb=c),   # shape
        lambda: tr.track(d, d, k, np.eye(4), init_nodes=n0, rgb=c.transpose(1, 2).contiguous().transpose(1, 2),
                         ref_rgb=c),                                                          # not contiguous
        lambda: tr.track(d, d, k, np.eye(4), init_nodes=n0),                                  # no rgb
        lambda: FrameTracker().track(d, d, k, np.eye(4), init_nodes=n0, rgb=c, ref_rgb=c),   # rgb, no term
        lambda: vol.raycast(k, np.eye(4), (24, 32), color=True),                              # colourless volume
        lambda: vol.raycast(k, np.eye(4), (24, 32), color=1),
    ]
    for call in calls:
        with pytest.raises((ValueError, _capi.OdbError)):
            call()
    assert _capi.launch_count() == n


def _track(tr, pred, ref_depth, ref, init, n0, rgb=None, ref_rgb=None):
    kw = dict(rgb=rgb, ref_rgb=ref_rgb) if tr.photometric > 0 else {}
    return tr.track(pred, ref_depth, K, ref, init, init_nodes=n0, **kw)


def test_textured_single_wall_against_exact_depth_and_colour():
    """Facing one wall, geometry alone is degenerate; with the texture the pose is recovered to the bounds of
    test_recovery_against_exact_geometry."""
    from omnidata_b200.track import STATUS, FrameTracker
    eye = np.array([0.0, 0.0, 0.0])
    kw = (400.0, 400.0, K[2], K[3])
    ref = VO.look_at(eye, eye + np.array([1.0, 0.0, 0.0]))
    far = (0.0, 0.0, -40.0)

    def scene(T):
        return (_t(VO.sphere_room_depth(kw, T, SIZE, far, 0.1, ROOM_LO, ROOM_HI).astype(np.float32)),
                _t(CO.sphere_room_rgb(kw, T, SIZE, far, 0.1, ROOM_LO, ROOM_HI).astype(np.float32)))

    d_ref, c_ref = scene(ref)
    for seed in range(3):
        rng = np.random.default_rng(300 + seed)
        truth = TO.perturb(ref, rng.uniform(0.0, 0.02), np.radians(rng.uniform(0.0, 1.5)), rng)
        d, c = scene(truth)
        _, _, rec = FrameTracker(affine=False).track(d, d_ref, kw, ref)
        assert STATUS[int(rec[1])] == "degenerate"
        pose, _, rec = FrameTracker(affine=False, photometric=LAMBDA, iterations=30).track(d, d_ref, kw, ref, rgb=c,
                                                                                           ref_rgb=c_ref)
        rec = rec.cpu().numpy()
        dp, dr = TO.pose_error(pose.cpu().numpy(), truth)
        print(f"textured wall, seed {seed}: {dp * 1e3:.3f} mm, {np.degrees(dr):.4f} deg, {int(rec[4])} iterations, "
              f"{int(rec[8])} photometric terms, RMS {rec[9]:.2e}")
        assert STATUS[int(rec[1])] == "ok" and dp < 2e-3 and dr < np.radians(0.1)


def test_weak_views_of_the_chained_path():
    """test_chained_tracking_against_exact_geometry with exact colour, geometry alone and with the term in the same
    run: the largest rotation error must fall below 0.2 degrees and below geometry alone's."""
    from omnidata_b200.track import FrameTracker
    path = TO.camera_path(48, CENTER, seed=3)
    errs = {}
    for lam in (0.0, LAMBDA):
        rng = np.random.default_rng(17)
        aligner, tr = _aligner(), FrameTracker(photometric=lam)
        last, e = path[0], []
        for T in path[1:]:
            s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
            pred = _t((s1 * _depth(T) + t1).astype(np.float32)).unsqueeze(0)
            ref = _t(_depth(last).astype(np.float32))
            n0, _ = aligner.fit(pred, ref.unsqueeze(0))
            pose, _, rec = _track(tr, pred, ref, last, None, n0.clone(), _t(_rgb(T)), _t(_rgb(last)))
            assert int(rec[1]) == 0
            last = pose.cpu().numpy()
            e.append(TO.pose_error(last, T))
        errs[lam] = np.array(e)
        print(f"chained, exact model, lambda {lam}: position max {errs[lam][:, 0].max() * 1e3:.3f} mm, rotation max "
              f"{np.degrees(errs[lam][:, 1].max()):.4f} deg (frame {int(np.argmax(errs[lam][:, 1])) + 1}), median "
              f"{np.degrees(np.median(errs[lam][:, 1])):.4f} deg")
    geo, photo = errs[0.0][:, 1].max(), errs[LAMBDA][:, 1].max()
    assert photo < np.radians(0.2) and photo < geo
    assert errs[LAMBDA][:, 0].max() < 1e-3


def test_frame_to_model_recovery_with_colour():
    """test_frame_to_model_recovery's bounds against a fused colour model, with the coloured raycast as ref_rgb."""
    from omnidata_b200.track import FrameTracker
    vol = _colour_volume(FINE)
    for seed in range(3):
        rng = np.random.default_rng(200 + seed)
        ref = TO.camera_path(1, CENTER, seed=seed)[0]
        off = rng.uniform(0.0, 0.05)
        truth = TO.perturb(ref, off, np.radians(rng.uniform(0.0, 3.0)), rng)
        s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        ref_depth, ref_rgb = vol.raycast(K, ref, SIZE, color=True)
        pred = _t((s1 * _depth(truth) + t1).astype(np.float32))
        nodes0, _ = _aligner().fit(pred.unsqueeze(0), ref_depth.unsqueeze(0))
        res = {}
        for lam in (0.0, LAMBDA):
            pose, nodes, rec = _track(FrameTracker(photometric=lam), pred, ref_depth, ref, None, nodes0.clone(),
                                      _t(_rgb(truth)), ref_rgb)
            assert int(rec[1]) == 0
            dp, dr = TO.pose_error(pose.cpu().numpy(), truth)
            res[lam] = (dp, dr, abs(float(nodes[0, 0, 0, 0]) * s1 - 1))
        print(f"fused colour model, seed {seed}: geometry {res[0.0][0] * 1e3:.3f} mm {np.degrees(res[0.0][1]):.4f} "
              f"deg; photometric {res[LAMBDA][0] * 1e3:.3f} mm {np.degrees(res[LAMBDA][1]):.4f} deg")
        dp, dr, ds = res[LAMBDA]
        assert dp < FINE / 4 and dp < 0.2 * off and dr < np.radians(0.5) and ds < 5e-3


def _path_run(path, voxel, size, f, noisy, seed, lam):
    """test_track_gpu._path_run with a colour volume and trackers with the given lambda."""
    import reconstruct
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    from test_track_gpu import _room_bounds_in
    rng = np.random.default_rng(seed)
    h, w = size
    k = (f, f, (w - 1) / 2, (h - 1) / 2)
    T0 = path[0] if noisy is None else np.eye(4)
    if noisy is None:
        origin, dims = _room_bounds_in(T0, voxel)
    else:
        n = int(round(3.2 / voxel)) + 1
        origin, dims = (-1.6, -1.6, -1.6), (n, n, n)
    vol = TSDFVolume(origin, voxel, dims, color=True, device=dev)
    aligner = _aligner()
    trackers = {a: FrameTracker(affine=a, photometric=lam) for a in (False, True)}
    last, errs, noise = np.eye(4), [], []
    for q, T in enumerate(path):
        truth = np.linalg.inv(T0) @ T
        d = _depth(T, size, k)
        rgb = _t(_rgb(T, size, k))
        s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        pred = _t((s1 * d + t1).astype(np.float32)).unsqueeze(0)
        if q == 0:
            sp = np.zeros(size, np.float32)
            idx = rng.choice(d.size, 300, replace=False)
            sp.reshape(-1)[idx] = d.reshape(-1)[idx]
            rec, _ = reconstruct.align_and_integrate(vol, aligner, pred, k, truth, _t(sp).unsqueeze(0), rgb)
            assert int(rec[1]) == 0
            continue
        init = last if noisy is None else TO.perturb(T, noisy[0], noisy[1], rng)
        noise.append(TO.pose_error(init, truth))
        failure, pose, _ = reconstruct.track_and_integrate(vol, aligner, trackers, pred, k, init, None, rgb)
        assert failure is None, (q, failure)
        last = pose
        errs.append(TO.pose_error(pose, truth))
    return np.array(errs), np.array(noise)


def test_unposed_reconstruction_with_colour():
    """test_unposed_reconstruction's bounds with the term; drift reported next to geometry alone's in the same run."""
    res = {lam: _path_run(TO.camera_path(48, CENTER, seed=3), FINE, SIZE, F, None, 17, lam)[0]
           for lam in (0.0, LAMBDA)}
    for lam, errs in res.items():
        print(f"unposed, colour volume, lambda {lam}: position error max {errs[:, 0].max() * 1e3:.2f} mm (last "
              f"{errs[-1, 0] * 1e3:.2f}), rotation max {np.degrees(errs[:, 1].max()):.3f} deg")
    errs = res[LAMBDA]
    assert errs[:, 0].max() < 2 * FINE and errs[:, 1].max() < np.radians(1.0)


def test_pose_refinement_with_colour():
    """test_pose_refinement's bounds with the term; reported next to geometry alone in the same run."""
    res = {lam: _path_run(TO.camera_path(40, CENTER, seed=5), FINE, (240, 320), 2 * F, (0.02, np.radians(1.5)), 17,
                          lam) for lam in (0.0, LAMBDA)}
    for lam, (errs, noise) in res.items():
        print(f"refined, colour volume, lambda {lam}: position error max {errs[:, 0].max() * 1e3:.2f} mm, mean "
              f"{errs[:, 0].mean() * 1e3:.2f} mm (input {noise[:, 0].mean() * 1e3:.1f} mm); rotation max "
              f"{np.degrees(errs[:, 1].max()):.3f} deg")
    errs, noise = res[LAMBDA]
    assert np.all(errs[:, 0] < noise[:, 0]) and errs[:, 0].mean() < 0.5 * noise[:, 0].mean()
    assert np.all(errs[:, 1] < noise[:, 1])


def test_reconstruct_cli_colour_and_photometric(tmp_path, capsys):
    """Runs end to end with random weights and no poses: a coloured PLY and one JSON line; no claim on quality."""
    import reconstruct
    from PIL import Image
    rng = np.random.default_rng(6)
    h = w = 384
    k = (300.0, 300.0, (w - 1) / 2, (h - 1) / 2)
    for sub in ("img", "sparse"):
        (tmp_path / sub).mkdir()
    for q, pose in enumerate(TO.camera_path(3, CENTER)):
        Image.fromarray(rng.integers(0, 255, (h, w, 3), dtype=np.uint8)).save(tmp_path / "img" / f"f{q}.png")
        if q == 0:
            d = VO.sphere_room_depth(k, pose, (h, w), CENTER, RADIUS, ROOM_LO, ROOM_HI)
            sp = np.zeros((h, w), np.uint16)
            idx = rng.choice(h * w, 500, replace=False)
            sp.reshape(-1)[idx] = np.rint(d.reshape(-1)[idx] * 1000).astype(np.uint16)
            Image.fromarray(sp).save(tmp_path / "sparse" / f"f{q}.png")
    out = tmp_path / "mesh.ply"
    res = reconstruct.main(["--img_path", str(tmp_path / "img"), "--intrinsics", ",".join(str(v) for v in k),
                            "--voxel", "0.05", "--bounds=-1.6,-1.6,0.1,1.6,1.6,3.3", "--out", str(out),
                            "--synthetic_weights", "--mode", "direct", "--sparse_path", str(tmp_path / "sparse"),
                            "--photometric", str(LAMBDA)])
    lines = capsys.readouterr().out.strip().splitlines()
    assert json.loads(lines[-1]) == res and res["frames"] == 3
    assert res["frames_used"] + len(res["frames_skipped"]) == 3
    header = out.read_bytes().split(b"end_header")[0].decode("ascii")
    assert "property uchar red" in header and f"element vertex {res['vertices']}" in header
