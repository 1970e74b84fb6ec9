"""MSDeformAttnPixelDecoder3D (CUDA, through the C ABI) vs the oracle port and the reference-generated golden fixture
(tests/golden/neck_small.npz, produced by oracle/gen_golden.py from the reference's own module under the shim).
Tolerance = SURVEY.md 8(d), both criteria (tests/util.py)."""
import pytest
import torch

from oracle import port
from util import assert_close, golden

pytestmark = pytest.mark.gpu


def _neck(cuda, c, sd):
    from occformer_b200.neck import MSDeformAttnPixelDecoder3D, neck_cfg
    n = MSDeformAttnPixelDecoder3D(**neck_cfg(c["in_channels"], c["strides"], c["E"], c["layers"], c["heads"], c["levels"],
                                              c["points"], c["ffn"]))
    n.load_state_dict(sd, strict=True)
    return n.to(cuda).eval()


@pytest.mark.parametrize("B", [1, 2])
def test_neck_vs_reference_golden_and_port(cuda, B):
    c = port.NECK_CASE
    sd = port.make_neck_state(c["in_channels"], c["E"], c["layers"], c["heads"], c["levels"], c["points"], c["ffn"],
                              seed=c["wseed"])
    feats = port.neck_inputs(c, B=B)
    neck = _neck(cuda, c, sd)
    outs = neck([f.to(cuda) for f in feats])
    want = port.ms_deform_pixel_decoder_3d(feats, sd, c["strides"], c["heads"], c["layers"], c["levels"], c["points"])
    assert len(outs) == len(want) == 4
    gold = golden("neck_small.npz")
    for i, (o, r) in enumerate(zip(outs, want)):
        assert o.shape == r.shape
        assert_close(o, r, what=f"neck out[{i}] {tuple(r.shape)} vs port (B={B})")
        if B == 1:
            assert_close(o, torch.from_numpy(gold[f"out{i}"]), what=f"neck out[{i}] vs reference golden")
    # the S32 twin handed to the head equals split(mask_feature)
    from occformer_b200 import ops
    from occformer_b200.common import twin_of
    mf = outs[0].permute(0, 2, 3, 4, 1).contiguous()
    assert torch.equal(ops.to_split(mf).view(torch.int32), twin_of(outs[0]).view(torch.int32))


def test_neck_full_width_pr1_grid(cuda):
    """The reference width (E = 192, 8 heads of 24, ffn 768, in_channels 128..1024, strides 2..16) on the PR1 pyramid
    (50x50x8 .. 7x7x1: odd sizes, non-divisible up-sampling ratios), 2 encoder layers."""
    c = dict(in_channels=[128, 256, 512, 1024], strides=[2, 4, 8, 16], E=192, layers=2, heads=8, levels=3, points=4, ffn=768,
             sizes=[(50, 50, 8), (25, 25, 4), (13, 13, 2), (7, 7, 1)], wseed=5, xseed=6)
    sd = port.make_neck_state(c["in_channels"], c["E"], c["layers"], c["heads"], c["levels"], c["points"], c["ffn"], seed=5)
    feats = port.neck_inputs(c, B=1)
    neck = _neck(cuda, c, sd)
    outs = neck([f.to(cuda) for f in feats])
    want = port.ms_deform_pixel_decoder_3d(feats, sd, c["strides"], c["heads"], c["layers"], c["levels"], c["points"])
    for i, (o, r) in enumerate(zip(outs, want)):
        assert_close(o, r, what=f"full-width neck out[{i}] {tuple(r.shape)}")
