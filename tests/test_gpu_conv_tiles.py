"""Conv tilings of occ_conv_bf16x3: 256-row tiles (MT = 2, two m64 chains per consumer warpgroup sharing each weight
k-block, per-warp epilogue staging) and the least-padding voxel boxes, vs fp64 torch at the 5e-5 gate of
test_gpu_gemm.py.  Every case first checks through occ_conv_plan that it runs the tiling it is meant to cover (the plan
depends on the SM count: these shapes are chosen for the 132 SMs of an H100 SXM)."""
import pytest
import torch
import torch.nn.functional as F

from util import assert_close

TOL = 5e-5

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape,plan", [
    # the bench's convs at batch 4: stage 0, neck output conv, stage 1 (s2 + s1), stage 2 (stays on 128-row tiles)
    ((4, 200, 200, 16, 128, 128, 1), (256, 128, 4, 1)),
    ((4, 200, 200, 16, 192, 192, 1), (256, 96, 4, 1)),
    ((4, 200, 200, 16, 128, 256, 2), (256, 128, 4, 1)),
    ((4, 100, 100, 8, 256, 256, 1), (256, 128, 4, 1)),
    ((4, 50, 50, 4, 512, 512, 1), (128, 128, 3, 1)),
])
def test_conv_plan(cuda, shape, plan):
    from occformer_b200 import ops
    B, X, Y, Z, Cin, Cout, stride = shape
    assert ops.conv_plan(B, X, Y, Z, Cin, Cout, stride=stride) == plan


CASES = [
    # B, X, Y, Z, Cin, Cout, stride, groups, plan
    (1, 101, 83, 16, 96, 128, 1, 32, (256, 128, 4, 1)),   # partial boxes along x and y
    (2, 140, 120, 32, 96, 128, 2, 32, (256, 128, 4, 1)),  # stride 2 (TMA element strides), two batch samples
    (1, 70, 64, 16, 96, 192, 1, 96, (256, 96, 4, 1)),     # the neck's sub-group statistics: cpg = 2, 96 groups
]


@pytest.mark.parametrize("case", CASES)
def test_conv_mt2(cuda, case):
    from occformer_b200 import ops
    B, X, Y, Z, Cin, Cout, stride, groups, plan = case
    assert ops.conv_plan(B, X, Y, Z, Cin, Cout, stride=stride) == plan
    g = torch.Generator().manual_seed(X + Y + Cout)
    x = torch.randn(B, Cin, X, Y, Z, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, 3, generator=g) * (27 * Cin) ** -0.5
    ref = F.conv3d(x.double(), w.double(), None, stride=stride, padding=1)
    w2, ks = ops.repack_conv_weight(w)
    w2 = w2.to(cuda)
    x_cl = ops.to_split(x.to(cuda).permute(0, 2, 3, 4, 1).contiguous())
    stats = torch.zeros((B, groups, 2), dtype=torch.float64, device=cuda)
    out = ops.conv(x_cl, w2, ks, stride=stride, gn_stats=stats, cpg=Cout // groups)
    assert_close(out.permute(0, 4, 1, 2, 3), ref, TOL, f"conv {case}")
    r = ref.reshape(B, groups, -1)
    assert_close(stats, torch.stack((r.sum(-1), (r * r).sum(-1)), dim=-1), 1e-4, f"conv gn_stats {case}")
    for _ in range(3):
        assert torch.equal(ops.conv(x_cl, w2, ks, stride=stride), out), f"conv {case} is not bit-reproducible"


def test_conv_mt2_epilogue(cuda):
    """bias + residual + activation + S32 output on 256-row tiles (never split-K)"""
    from occformer_b200 import ops
    B, X, Y, Z, Cin, Cout = 1, 101, 83, 16, 96, 128
    assert ops.conv_plan(B, X, Y, Z, Cin, Cout, splitk_ok=False) == (256, 128, 4, 1)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, Cin, X, Y, Z, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, 3, generator=g) * (27 * Cin) ** -0.5
    bias, res = torch.randn(Cout, generator=g), torch.randn(B, X, Y, Z, Cout, generator=g)
    ref = F.conv3d(x.double(), w.double(), bias.double(), padding=1).permute(0, 2, 3, 4, 1) + res.double()
    w2, ks = ops.repack_conv_weight(w)
    w2 = w2.to(cuda)
    x_cl = ops.to_split(x.to(cuda).permute(0, 2, 3, 4, 1).contiguous())
    out = ops.conv(x_cl, w2, ks, bias=bias.to(cuda), residual=res.to(cuda), act=1)
    assert_close(out, F.relu(ref), TOL, "conv MT2 epilogue")
    out_s = ops.conv(x_cl, w2, ks, bias=bias.to(cuda), residual=res.to(cuda), act=1, split_out=True)
    assert torch.equal(out_s.view(torch.int32), ops.to_split(out).view(torch.int32)), "split_out != split(out)"
