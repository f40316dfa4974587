"""Host-side checks of the normal-model train step that run before any engine or launch exists: each train step refuses a
model of the other task, and NormalStepLoss refuses mis-shaped tensors."""
import pytest
import torch


def _model(num_channels):
    from omnidata_b200.model import DPTDepthModel
    return DPTDepthModel(backbone="vitb_rn50_384", num_channels=num_channels)


def test_each_train_step_refuses_the_other_tasks_model():
    from omnidata_b200.train import DepthTrainStep, NormalTrainStep
    with pytest.raises(ValueError, match="num_channels"):
        DepthTrainStep(_model(3))
    with pytest.raises(ValueError, match="num_channels"):
        NormalTrainStep(_model(1))


@pytest.mark.parametrize("pred,gt,mask", [
    ((2, 1, 64, 64), (2, 1, 64, 64), (2, 1, 64, 64)),        # a depth-shaped prediction
    ((2, 3, 64, 64), (2, 3, 64, 96), (2, 1, 64, 64)),        # target of another size
    ((2, 3, 64, 64), (1, 3, 64, 64), (2, 1, 64, 64)),        # target of another batch
    ((2, 3, 64, 64), (2, 3, 64, 64), (2, 3, 64, 64)),        # the reference's repeated mask instead of mask_float
    ((2, 3, 64, 64), (2, 3, 64, 64), (2, 64, 64)),           # mask without its channel axis
    ((3, 64, 64), (3, 64, 64), (1, 64, 64)),                 # no batch axis
])
def test_normal_step_loss_rejects_wrong_shapes(pred, gt, mask):
    from omnidata_b200.losses import NormalStepLoss
    with pytest.raises(ValueError):
        NormalStepLoss()(torch.zeros(pred), torch.zeros(gt), torch.zeros(mask))
