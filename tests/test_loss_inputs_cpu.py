"""render_loss_batch validates the image-loss tensors it hands to the fused loss kernel (csrc/loss.cu) before any device
work: shapes first, then devices.  The kernel reads them as raw (M,3,H,W) / (M,H,W) / (3,) buffers on the rasterizer's
device, so a (H,W) mask for M > 1 frames or a host tensor would otherwise be read past its end."""
import types

import pytest
import torch

M, H, W = 3, 20, 36
CUDA0 = torch.device("cuda", 0)


class _OnDevice:
    """Shape and device of a tensor on a CUDA device, for a machine that has none."""

    def __init__(self, *shape, device=CUDA0):
        self.shape, self.device, self.is_cuda = torch.Size(shape), device, True

    def numel(self):
        return self.shape.numel()


def _check(**kw):
    from vidu4d_b200.renderer import _check_loss_inputs
    args = dict(target_rgb=_OnDevice(M, 3, H, W), vis2d=None, mask_gt=None, mask_wt=None, learnable_bkgd=None)
    args.update(kw)
    _check_loss_inputs(M, H, W, CUDA0, **args)


@pytest.mark.parametrize("kw,msg", [
    (dict(target_rgb=torch.zeros(3, H, W)), r"target_rgb must be \(M,3,H,W\) = \(3,3,20,36\), got \(3, 20, 36\)"),
    (dict(target_rgb=torch.zeros(M, 3, W, H)), r"target_rgb must be .* got \(3, 3, 36, 20\)"),
    (dict(target_rgb=torch.zeros(M, 4, H, W)), r"target_rgb must be .* got \(3, 4, 20, 36\)"),
    (dict(vis2d=torch.zeros(H, W)), r"vis2d must be \(M,H,W\) = \(3,20,36\) or None, got \(20, 36\)"),
    (dict(mask_gt=torch.zeros(M, 1, H, W)), r"mask_gt must be \(M,H,W\) .* got \(3, 1, 20, 36\)"),
    (dict(mask_gt=torch.zeros(M, H, W), mask_wt=torch.zeros(1, H, W)), r"mask_wt must be \(M,H,W\) .* got \(1, 20, 36\)"),
    (dict(mask_wt=torch.zeros(M, H, W)), r"mask_wt weights the mask term: it needs mask_gt"),
    (dict(learnable_bkgd=torch.zeros(4)), r"learnable_bkgd must have 3 elements, got shape \(4,\)"),
    (dict(learnable_bkgd=torch.zeros(M, 3)), r"learnable_bkgd must have 3 elements, got shape \(3, 3\)"),
])
def test_wrong_shapes_are_refused(kw, msg):
    with pytest.raises(RuntimeError, match=msg):
        _check(**kw)


def test_shapes_are_checked_before_devices():
    # a host tensor of the wrong shape reports its shape, not its device
    with pytest.raises(RuntimeError, match="vis2d must be"):
        _check(vis2d=torch.zeros(M * H * W))


@pytest.mark.parametrize("name", ["target_rgb", "vis2d", "mask_gt", "mask_wt", "learnable_bkgd"])
def test_host_tensors_are_refused(name):
    shape = {"target_rgb": (M, 3, H, W), "learnable_bkgd": (3,)}.get(name, (M, H, W))
    kw = {name: torch.zeros(shape)}
    if name == "mask_wt":
        kw["mask_gt"] = _OnDevice(M, H, W)
    with pytest.raises(RuntimeError, match=f"{name} must be a CUDA tensor on the rasterizer's device cuda:0, got cpu"):
        _check(**kw)
    kw[name] = _OnDevice(*shape, device=torch.device("cuda", 1))       # another GPU than the rasterizer's
    with pytest.raises(RuntimeError, match=f"{name} must be a CUDA tensor on the rasterizer's device cuda:0, got cuda:1"):
        _check(**kw)


def test_well_formed_inputs_pass():
    _check(vis2d=_OnDevice(M, H, W), mask_gt=_OnDevice(M, H, W), mask_wt=_OnDevice(M, H, W), learnable_bkgd=_OnDevice(3))
    _check(mask_gt=_OnDevice(M, H, W), learnable_bkgd=_OnDevice(1, 3))


def test_render_loss_batch_refuses_before_touching_the_device():
    """Through the public entry point, with host tensors everywhere: the validation error comes first."""
    from vidu4d_b200.renderer import BatchCameras, PipelineParams, render_loss_batch
    cams = BatchCameras(W, H, 1.0, 0.8, torch.eye(4).repeat(M, 1, 1), torch.eye(4).repeat(M, 1, 1), torch.zeros(M, 3))
    pc = types.SimpleNamespace(get_xyz=torch.zeros(10, 3), get_rotation=torch.zeros(10, 4), active_sh_degree=0)
    with pytest.raises(RuntimeError, match="mask_gt must be"):
        render_loss_batch(cams, pc, PipelineParams(), torch.zeros(3), torch.zeros(M, 3, H, W), mask_gt=torch.zeros(H, W))
    with pytest.raises(RuntimeError, match="target_rgb must be a CUDA tensor"):
        render_loss_batch(cams, pc, PipelineParams(), torch.zeros(3), torch.zeros(M, 3, H, W))
