"""Host-side checks that keep the VNL kernels' unchecked gathers in bounds (no device needed: they run before any launch)."""
import numpy as np
import pytest
import torch


def test_vnl_points_are_checked_against_the_prediction_size():
    from omnidata_b200.losses import VNL_Loss, check_vnl_points
    np.random.seed(0)
    pts = VNL_Loss(1.0, 1.0, (320, 480)).select_index()
    check_vnl_points(pts, 320, 480)
    check_vnl_points([torch.from_numpy(p) for p in pts], 320, 480)                  # host tensors are read as well
    with pytest.raises(ValueError):
        check_vnl_points(pts, 256, 256)                                             # drawn over a larger image
    for i, v in ((0, -1), (2, 320 * 480)):
        bad = [p.copy() for p in pts]
        bad[i][5] = v
        with pytest.raises(ValueError):
            check_vnl_points(bad, 320, 480)
    with pytest.raises(ValueError):
        check_vnl_points([pts[0], pts[1][:-1], pts[2]], 320, 480)                   # unequal lengths
    with pytest.raises(ValueError):
        check_vnl_points(pts[:2], 320, 480)


def test_depth_step_loss_rejects_another_size():
    from omnidata_b200.losses import DepthStepLoss
    fn = DepthStepLoss((320, 480))
    t = torch.zeros(2, 1, 384, 384)
    with pytest.raises(ValueError):
        fn(t, t, t, full_mix=False)
