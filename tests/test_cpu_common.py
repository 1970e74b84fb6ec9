"""The package's module conventions (occformer_b200/common.py) on the CPU: the rule by which a module picks up the S32
twin of its input, the prepared-parameter cache of every module that runs on the kernels, and the view transformer's
host copy of its grid."""
import pytest
import torch

from occformer_b200.common import attach_twin, twin_of
from occformer_b200.depthnet import DepthNet
from occformer_b200.efficientnet import CustomEfficientNet
from occformer_b200.encoder import DualpathTransformerBlock
from occformer_b200.head import Mask2FormerNuscOccHead, head_cfg
from occformer_b200.image_encoder import ResNet
from occformer_b200.neck import MSDeformAttnPixelDecoder3D, neck_cfg
from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel


def _handed_over(*shape, C=64, Cp=None):
    """(channel-last base (n, *spatial, Cp), its (n, C, *spatial) view as a module returns it, a twin of the base's
    shape) -- the twin's values do not matter to the rule"""
    g = torch.Generator().manual_seed(0)
    base = torch.randn(*shape, Cp or C, generator=g)
    view = base[..., :C].permute(0, base.dim() - 1, *range(1, base.dim() - 1))
    return base, view, torch.randn(base.shape, generator=g)


# ------------------------------------------------------------------ the twin rule
@pytest.mark.parametrize("shape", [(2, 4, 6), (2, 4, 6, 3)], ids=["image", "voxel"])
def test_twin_accepted_while_unmodified(shape):
    _, v, s = _handed_over(*shape)
    assert attach_twin(v, s) is v
    assert twin_of(v) is s
    assert twin_of(v.float()) is s  # .float() of an fp32 tensor is the tensor itself


@pytest.mark.parametrize("change", ["view", "base", "other view"])
def test_twin_rejected_after_in_place_change(change):
    base, v, s = _handed_over(2, 4, 6)
    attach_twin(v, s)
    if change == "view":
        v.mul_(2)
    elif change == "base":
        base.relu_()
    else:
        base[0, 0].zero_()
    assert twin_of(v) is None


def test_twin_rejected_when_it_does_not_match():
    _, v, s = _handed_over(2, 4, 6)
    assert twin_of(v) is None  # nothing attached
    v._occ_s32 = s  # set by hand, without attach_twin's stamp
    assert twin_of(v) is None
    for bad in (s[..., :32], s.double(), s.permute(0, 2, 1, 3), torch.empty(s.shape, device="meta")):
        assert twin_of(attach_twin(v, bad)) is None
    assert twin_of(attach_twin(v, s)) is s


def test_zero_padded_twin_of_a_narrow_level():
    """a 48-wide stage as CustomEfficientNet hands it over: its twin is padded to 64 columns"""
    _, v, s = _handed_over(2, 4, 6, C=48, Cp=64)
    assert v.shape == (2, 48, 4, 6)
    assert twin_of(attach_twin(v, s)) is s
    assert twin_of(attach_twin(v, s[..., :48])) is None


def test_twin_of_an_inference_tensor():
    """inference tensors have no version counter: the twin is accepted, also after an in-place change"""
    with torch.inference_mode():
        _, v, s = _handed_over(2, 4, 6)
        attach_twin(v, s)
    assert v.is_inference() and twin_of(v) is s
    with torch.inference_mode():
        v.mul_(2)
    assert twin_of(v) is s
    _, w, s2 = _handed_over(2, 4, 6)
    attach_twin(w, s2)
    w._occ_s32_version = None  # an inference tensor's stamp on an ordinary tensor
    assert twin_of(w) is None


# ------------------------------------------------------------------ the prepared-parameter cache
# SECONDFPN, the eighth, is covered by tests/test_cpu_image_encoder.py::test_prepare_cache_dropped_by_load_state_dict
MODULES = {
    "ResNet": lambda: ResNet(50, num_stages=1, strides=(1,), dilations=(1,), out_indices=(0,)),
    "CustomEfficientNet": lambda: CustomEfficientNet("b0", out_indices=(2, 3)),
    "DepthNet": lambda: DepthNet(32, 64, 16, 8, cam_channels=27),
    "DualpathTransformerBlock": lambda: DualpathTransformerBlock(128, 128, norm_cfg=dict(type="GN", num_groups=32),
                                                                 layer_index=0),
    "MSDeformAttnPixelDecoder3D": lambda: MSDeformAttnPixelDecoder3D(**neck_cfg([32, 64, 64, 64], [2, 4, 8, 16], 64, 1,
                                                                                2, 3, 4, 128)),
    "Mask2FormerOccHead": lambda: Mask2FormerNuscOccHead(**head_cfg(96, 8, 5, 1, 3, [-1.0, -1.0, -1.0, 1.0, 1.0, 1.0])),
    "ViewTransformerLiftSplatShootVoxel": lambda: ViewTransformerLiftSplatShootVoxel(numC_input=64, numC_Trans=32),
}


@pytest.mark.parametrize("name", list(MODULES))
def test_prepare_cache_dropped_by_load_state_dict_and_to(name):
    net = MODULES[name]().eval()
    net._prep = object()
    net.load_state_dict(net.state_dict())
    assert net._prep is None
    net._prep = object()
    net.double()
    assert net._prep is None


def test_view_transformer_grid_follows_load_state_dict():
    vt = ViewTransformerLiftSplatShootVoxel(numC_input=64, numC_Trans=32)
    assert vt.grid_size() == (128, 128, 1)
    assert vt.prepared() is vt.prepared()
    sd = vt.state_dict()
    sd["nx"] = sd["nx"] * 2
    sd["dx"] = sd["dx"] / 2
    vt.load_state_dict(sd)
    assert vt.grid_size() == (256, 256, 2)
    assert vt.prepared() == (vt.dx.tolist(), vt.bx.tolist(), vt.nx.tolist())
