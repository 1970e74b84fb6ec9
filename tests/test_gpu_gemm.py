"""wgmma split-bf16 (three-pass, fp32-faithful) GEMM / implicit-GEMM conv vs fp64 torch on arbitrary fp32 operands.
Expected error: ~4e-6 rms / ~2e-5 worst case relative (dropped lo*lo term + hi/lo roundings, <= 3 * 2^-18 per product);
gate 5e-5 on both SURVEY criteria -- 20x inside the 1e-3 north-star tolerance."""
import pytest
import torch
import torch.nn.functional as F

from util import assert_close

TOL = 5e-5

pytestmark = pytest.mark.gpu


def _mk(shape, g, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


def test_split_roundtrip(cuda):
    """S32 format: device split == torch split (ops.split_weight), unsplit(split(x)) == x to 2^-17 relative."""
    from occformer_b200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn(257, 160, generator=g) * torch.logspace(-3, 3, 160)
    xs = ops.to_split(x.to(cuda))
    assert torch.equal(xs.cpu().view(torch.int32), ops.split_weight(x).view(torch.int32)), "device / host split differ"
    back = ops.from_split(xs).cpu()
    assert float(((back - x).abs() / x.abs().clamp_min(1e-30)).max()) < 2 ** -16
    assert torch.equal(ops.unsplit_weight(xs.cpu()), back)


@pytest.mark.parametrize("M,N,K", [(300, 384, 128), (1000, 100, 192), (129, 18, 96), (128, 32, 32), (4096, 256, 256),
                                   (777, 1024, 512), (100, 1536, 192), (100, 192, 1536), (5000, 64, 160)])
def test_gemm_plain(cuda, M, N, K):
    from occformer_b200 import ops
    g = torch.Generator().manual_seed(M + N + K)
    a, w = _mk((M, K), g), _mk((N, K), g, K ** -0.5)
    out = ops.gemm(ops.to_split(a.to(cuda)), ops.split_weight(w).to(cuda))
    ref = a.double() @ w.double().t()
    assert_close(out, ref, TOL, f"gemm {M}x{N}x{K}")


@pytest.mark.parametrize("act", [0, 1, 2])
def test_gemm_epilogue(cuda, act):
    from occformer_b200 import ops
    g = torch.Generator().manual_seed(act)
    M, N, K = 1500, 384, 128
    a, w = _mk((M, K), g), _mk((N, K), g, K ** -0.5)
    bias, res = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    a_s, w_s = ops.to_split(a.to(cuda)), ops.split_weight(w).to(cuda)
    out = ops.gemm(a_s, w_s, bias=bias.to(cuda), residual=res.to(cuda), act=act)
    ref = a.double() @ w.double().t() + bias.double() + res.double()
    ref = [lambda x: x, F.relu, F.gelu][act](ref)
    assert_close(out, ref, TOL, f"gemm epilogue act={act}")
    # split_out: the epilogue writes the S32 format directly (operand of the next contraction) == split(fp32 output)
    plain = ops.gemm(a_s, w_s, bias=bias.to(cuda))
    out_s = ops.gemm(a_s, w_s, bias=bias.to(cuda), split_out=True)
    assert torch.equal(out_s.view(torch.int32), ops.to_split(plain).view(torch.int32)), "split_out != split(out)"


CONV_CASES = [
    # B, X, Y, Z, Cin, Cout, k, stride, dil
    (2, 15, 10, 4, 32, 64, (3, 3, 3), 1, 1),
    (1, 15, 10, 4, 64, 128, (3, 3, 3), 2, 1),
    (2, 9, 16, 2, 32, 32, (1, 1, 1), 2, 1),
    (1, 50, 50, 8, 128, 128, (3, 3, 3), 1, 1),
    (2, 25, 25, 1, 32, 32, (3, 3, 1), 1, 6),
    (1, 30, 20, 1, 64, 64, (3, 3, 1), 1, 18),
    (1, 7, 5, 3, 32, 256, (3, 3, 3), 2, 1),
    (1, 13, 13, 1, 160, 32, (1, 1, 1), 1, 1),
    # few output tiles, long K: split-K (partial sums meet through TMA reduce-add, GroupNorm statistics from the result)
    (1, 25, 25, 4, 256, 512, (3, 3, 3), 1, 1),
    (2, 50, 50, 8, 128, 256, (3, 3, 3), 2, 1),
    # many M-tiles, short K: 611 128-row tiles (1 x 4 x 32 voxel boxes) at BN 64, more than four per SM (27 k-blocks
    # and BN 64 keep it off the 256-row tiles, which need BN 96 / 128 and at least 64 k-blocks)
    (1, 47, 51, 32, 32, 64, (3, 3, 3), 1, 1),
    # group sizes that are not powers of two: 192 channels / 32 groups (cpg 6) in the epilogue, 96 / 32 (cpg 3) split-K
    (1, 20, 20, 4, 64, 192, (3, 3, 3), 1, 1),
    (1, 25, 25, 4, 256, 96, (3, 3, 3), 1, 1),
]
SPLITK_CASES = [CONV_CASES[8], CONV_CASES[9], CONV_CASES[12]]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv(cuda, case):
    from occformer_b200 import ops
    B, X, Y, Z, Cin, Cout, k, stride, dil = case
    g = torch.Generator().manual_seed(sum(case[:6]))
    x = _mk((B, Cin, X, Y, Z), g)
    w = _mk((Cout, Cin) + k, g, (Cin * k[0] * k[1] * k[2]) ** -0.5)
    pad = tuple(dil * (kk - 1) // 2 for kk in k)
    ref = F.conv3d(x.double(), w.double(), None, stride=stride, padding=pad, dilation=dil)
    w2, ks = ops.repack_conv_weight(w)
    w2 = w2.to(cuda)
    groups = 32 if (Cout == 32 and Cin == 160) else (16 if Cout == 32 else 32)  # covers cpg = 1, 2, 3, 4, 6, 8, 16
    if case in SPLITK_CASES:
        assert ops.conv_plan(B, X, Y, Z, Cin, Cout, k, stride, dil)[3] > 1, f"conv {case} does not run split-K"
    stats = torch.zeros((B, groups, 2), dtype=torch.float64, device=cuda)
    x_cl = ops.to_split(x.to(cuda).permute(0, 2, 3, 4, 1).contiguous())
    out = ops.conv(x_cl, w2, ks, stride=stride, dil=dil, gn_stats=stats, cpg=Cout // groups)
    assert_close(out.permute(0, 4, 1, 2, 3), ref, TOL, f"conv {case}")
    # GroupNorm statistics accumulated in the epilogue: (sum, sumsq) per (batch, group)
    r = ref.reshape(B, groups, -1)
    ref_stats = torch.stack((r.sum(-1), (r * r).sum(-1)), dim=-1)
    assert_close(stats, ref_stats, 1e-4, f"conv gn_stats {case}")  # tensor-core accumulation rounds toward zero
    # bit-reproducible, also on the split-K path (the splits add their partial sums in a fixed order)
    for _ in range(3):
        again = ops.conv(x_cl, w2, ks, stride=stride, dil=dil)
        assert torch.equal(again, out), f"conv {case} is not bit-reproducible"


def test_gemm_rejects_bad_args(cuda):
    from occformer_b200 import ops
    a = torch.zeros(8, 48, device=cuda)  # K % 32 != 0: not a whole number of S32 chunks
    w = torch.zeros(16, 48, device=cuda)
    with pytest.raises(RuntimeError):
        ops.gemm(a, w)
    with pytest.raises(RuntimeError):
        ops.gemm(torch.zeros(8, 32), torch.zeros(16, 32))  # CPU tensors: no fallback
    # GroupNorm statistics of more than 96 groups do not fit the epilogue's partial sums
    x = ops.to_split(torch.zeros(1, 4, 4, 4, 32, device=cuda))
    stats = torch.zeros(1, 128, 2, dtype=torch.float64, device=cuda)
    with pytest.raises(RuntimeError):
        ops.conv(x, torch.zeros(128, 32, device=cuda), (1, 1, 1), gn_stats=stats, cpg=1)


@pytest.mark.parametrize("B,X,Y,ch", [(1, 50, 50, 32), (2, 25, 30, 32), (1, 20, 20, 64)])
def test_conv_taps_merged_aspp_branches(cuda, B, X, Y, ch):
    """occ_conv_taps_bf16x3: the four ASPP branches (1x1 + 3x3 dilated 6 / 12 / 18, same input) as one 25-tap launch vs
    four torch convolutions; GroupNorm statistics of the 4 x groups from the epilogue."""
    from occformer_b200 import ops
    g = torch.Generator().manual_seed(X + ch)
    x = torch.randn(B, ch, X, Y, generator=g)
    dil = (1, 6, 12, 18)
    ws = [torch.randn(ch, ch, 1, 1, generator=g) * ch ** -0.5] + [torch.randn(ch, ch, 3, 3, generator=g) * (9 * ch) ** -0.5
                                                                 for _ in range(3)]
    ref = torch.cat([F.conv2d(x.double(), w.double(), padding=0 if w.shape[-1] == 1 else d, dilation=d)
                     for w, d in zip(ws, dil)], 1)
    taps = [(0, 0, 0)]
    for d in dil[1:]:
        taps += [(i * d, j * d, 0) for i in (-1, 0, 1) for j in (-1, 0, 1) if (i, j) != (0, 0)]
    wm = torch.zeros(4 * ch, len(taps), ch)
    wm[:ch, 0] = ws[0][:, :, 0, 0]
    for bi, d in enumerate(dil[1:], start=1):
        for i in (-1, 0, 1):
            for j in (-1, 0, 1):
                t = 0 if (i, j) == (0, 0) else taps.index((i * d, j * d, 0))
                wm[bi * ch:(bi + 1) * ch, t] = ws[bi][:, :, i + 1, j + 1]
    groups = 4 * (ch // 2)
    if groups > 64:
        groups = 64
    cpg = 4 * ch // groups
    stats = torch.zeros(B, groups, 2, dtype=torch.float64, device=cuda)
    xs = ops.to_split(x.permute(0, 2, 3, 1).contiguous().to(cuda)).view(B, X, Y, 1, ch)
    out = ops.conv_taps(xs, ops.split_weight(wm.reshape(4 * ch, -1)).to(cuda), taps, gn_stats=stats, cpg=cpg)
    assert_close(out.view(B, X, Y, 4 * ch).permute(0, 3, 1, 2), ref, TOL, f"merged ASPP branches {X}x{Y} ch={ch}")
    r = ref.reshape(B, groups, -1)
    assert_close(stats, torch.stack((r.sum(-1), (r * r).sum(-1)), -1), 1e-4, "merged ASPP gn_stats")
