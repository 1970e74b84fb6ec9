"""DepthNet on the library's kernels (depthnet.py _forward_cuda) and the launches it adds: the conv into a column slice,
the camera-aware SE gates, their application, the deformable im2col, the whole module and the view transformer that
runs it.  The oracle is depthnet.py's torch forward on the host in float64 (pinned to the reference class by
test_depthnet_vs_reference_golden) and the plain restatements of tests/depthnet_ref.py."""
import pytest
import torch
import torch.nn.functional as F

from depthnet_ref import cam_gates, deform_cols, group_cols
from util import assert_close, f64, parity_log, rel_err, run_trace
from vt_chain import check_pooled, config_view_transformer
from occformer_b200 import ops, synth
from occformer_b200.common import twin_of
from occformer_b200.depthnet import DepthNet

pytestmark = pytest.mark.gpu

KERNEL_TOL = 5e-5


def _unsplit(t):
    return ops.unsplit_weight(t.reshape(-1, t.shape[-1])).view(t.shape)


def _net(cin, mid, ctx, D, cam, seed, dev):
    net = DepthNet(cin, mid, ctx, D, cam_channels=cam).eval()
    net.load_state_dict(synth.make_depthnet_state(cin, mid, ctx, D, cam, seed=seed), strict=True)
    return net.to(dev)


# ------------------------------------------------------------------ 1. conv into a column slice
def _conv_case(dev, Cin, Cout, k, dil=1, seed=0, n=2, H=9, W=13):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) * (k * k * Cin) ** -0.5
    b = 0.1 * torch.randn(Cout, generator=g)
    x_s = ops.to_split(x.permute(0, 2, 3, 1).contiguous().to(dev)).view(n, H, W, 1, Cin)
    w2, ks = ops.repack_conv_weight(w.to(dev))
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=dil * (k // 2), dilation=dil)
    return x_s, w2, ks, b.to(dev), ref.permute(0, 2, 3, 1).reshape(-1, Cout)


SENTINEL = -1234.5


@pytest.mark.parametrize("Cout,ldo,off,k,dil,split", [
    (64, 160, 32, 3, 1, False),     # fp32, TMA store
    (112, 240, 0, 1, 1, False),     # fp32, DepthNet's depth head slice
    (128, 240, 112, 1, 1, False),   # fp32, DepthNet's context slice
    (18, 36, 8, 3, 1, False),       # fp32, Cout % 4 != 0: scalar stores
    (64, 160, 64, 3, 6, True),      # S32 slice, dilated
    (96, 320, 224, 1, 1, True),     # S32 slice at the end of the row
])
def test_conv_slice_against_fp64(cuda, Cout, ldo, off, k, dil, split):
    x_s, w2, ks, b, ref = _conv_case(cuda, 64, Cout, k, dil)
    rows = ref.shape[0]
    out = torch.full((rows, ldo), SENTINEL, device=cuda)
    ops.conv_into(x_s, w2, ks, out, off, dil=dil, bias=b, split_out=split)
    sl = out[:, off:off + Cout]
    got = _unsplit(sl.contiguous()) if split else sl
    r = assert_close(got, ref, KERNEL_TOL, f"conv slice Cout={Cout} ldo={ldo} off={off} split={split}")
    parity_log(f"[depthnet] conv slice Cout={Cout} ldo={ldo} off={off} split={int(split)}: rel_max {r:.2e}")
    outside = torch.cat([out[:, :off], out[:, off + Cout:]], dim=1)
    assert bool((outside.view(torch.int32) == torch.tensor(SENTINEL).view(torch.int32).item()).all()), \
        "columns outside the slice changed"
    # the same conv through occ_conv_bf16x3 (contiguous output) gives the same bits
    full = ops.conv(x_s, w2, ks, dil=dil, bias=b, split_out=split).view(rows, Cout)
    assert torch.equal(full.view(torch.int32), sl.contiguous().view(torch.int32))


def test_conv_full_width_slice_equals_conv(cuda):
    """occ_conv_slice_bf16x3 with ldo = Cout, out_off = 0 is occ_conv_bf16x3, bit for bit, at a shape that tiles with
    256-row tiles and at one with 128-row tiles"""
    for n, H, W, Cin, Cout in ((4, 16, 44, 256, 128), (1, 8, 12, 64, 64)):
        x_s, w2, ks, b, _ = _conv_case(cuda, Cin, Cout, 3, n=n, H=H, W=W)
        a = ops.conv(x_s, w2, ks, bias=b, act=1)
        out = torch.empty((n * H * W, Cout), device=cuda)
        ops.conv_into(x_s, w2, ks, out, 0, bias=b, act=1)
        assert torch.equal(a.view(-1, Cout), out)


def test_residual_is_added_before_the_activation(cuda):
    """gemm and conv compute act(A W^T + bias + residual): BasicBlock's relu(bn2(conv2) + identity)"""
    g = torch.Generator().manual_seed(5)
    M, K, N = 300, 64, 96
    a, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * K ** -0.5
    b, r = 0.1 * torch.randn(N, generator=g), 2.0 * torch.randn(M, N, generator=g)
    out = ops.gemm(ops.to_split(a.to(cuda)), ops.split_weight(w).to(cuda), bias=b.to(cuda), residual=r.to(cuda), act=1)
    pre = a.double() @ w.double().T + b.double()
    want = torch.relu(pre + r.double())
    assert_close(out, want, KERNEL_TOL, "gemm relu(x W^T + b + residual)")
    other = torch.relu(pre) + r.double()
    assert rel_err(want, other) > 0.1  # the two orders differ: the check above distinguishes them
    x_s, w2, ks, bb, ref = _conv_case(cuda, 64, 64, 3, seed=6)
    res = 2.0 * torch.randn(ref.shape, generator=g)
    y = ops.conv(x_s, w2, ks, bias=bb, residual=res.to(cuda), act=1).view(ref.shape)
    assert_close(y, torch.relu(ref + res.double()), KERNEL_TOL, "conv relu(conv + b + residual)")


# ------------------------------------------------------------------ 2. camera-aware gates
@pytest.mark.parametrize("cam,C", [(27, 512), (33, 640)])
def test_cam_gates_against_fp64(cuda, cam, C):
    net = _net(64, C, 32, 16, cam, 7, cuda)
    g = torch.Generator().manual_seed(8)
    m = torch.randn(6, cam, generator=g)
    P = net._prepare()
    gates = ops.depthnet_cam_gates(m.to(cuda), *P["gates"])
    want = cam_gates(m.double(), [t.double().cpu() for t in net._folded()["gates"]])
    r = assert_close(gates, want, KERNEL_TOL, f"cam gates cam={cam} C={C}")
    parity_log(f"[depthnet] cam gates cam={cam}: rel_max {r:.2e}")
    # against the module's own Mlp / SELayer chain (BatchNorm1d not folded), fp64
    ref = f64(net)
    with torch.no_grad():
        mm = ref.bn(m.double())
        for i, (mlp, se) in enumerate(((ref.depth_mlp, ref.depth_se), (ref.context_mlp, ref.context_se))):
            x_se = mlp(mm)[..., None, None]
            gd = se.gate(se.conv_expand(se.act1(se.conv_reduce(x_se))))[:, :, 0, 0]
            assert_close(gates[i], gd, KERNEL_TOL, f"cam gates chain {i} vs Mlp + SELayer")


# ------------------------------------------------------------------ 3. SE apply
def test_se_apply_bitwise(cuda):
    g = torch.Generator().manual_seed(9)
    n, HW, C = 6, 704, 512
    x = torch.randn(n * HW, C, generator=g).to(cuda)
    gates = torch.rand(2, n, C, generator=g).to(cuda)
    xd, xd_s, xc_s = ops.se_apply(x, gates, n, HW)
    wd = (x.view(n, HW, C) * gates[0].view(n, 1, C)).view(-1, C)
    wc = (x.view(n, HW, C) * gates[1].view(n, 1, C)).view(-1, C)
    assert torch.equal(xd.view(torch.int32), wd.view(torch.int32))
    assert torch.equal(xd_s.view(torch.int32), ops.to_split(wd).view(torch.int32))
    assert torch.equal(xc_s.view(torch.int32), ops.to_split(wc).view(torch.int32))


# ------------------------------------------------------------------ 4. deformable im2col
def _im2col_case(cuda, x, off, groups=4):
    n, C, H, W = x.shape
    x_s = ops.to_split(x.permute(0, 2, 3, 1).contiguous().to(cuda))
    off_cl = torch.zeros(n * H * W, 32)
    off_cl[:, :18] = off.permute(0, 2, 3, 1).reshape(-1, 18)
    cols = ops.deform_im2col(x_s, off_cl.to(cuda), n, H, W, groups)
    x_seen = _unsplit(x_s).cpu().view(n, H, W, C).permute(0, 3, 1, 2).double()
    want = group_cols(deform_cols(x_seen, off), groups)  # positions in fp32 as the kernel's, samples in fp64
    return _unsplit(cols), want


def test_deform_im2col_exact_positions(cuda):
    """Offsets on a 1/8 grid (every floor decision exact) and inputs k/8: every sample is exact in fp32 and S32.  Cases:
    integer positions, h exactly -1 / H-1 / H, h in (-1, 0), far outside."""
    n, C, H, W = 2, 128, 7, 10
    g = torch.Generator().manual_seed(10)
    x = torch.randint(-64, 65, (n, C, H, W), generator=g).float() / 8
    off = torch.randint(-24, 25, (n, 18, H, W), generator=g).float() / 8  # [-3, 3] in steps of 1/8
    off[:, 0, 0, :] = 0.0      # k = 0 at y = 0: h = -1 exactly (no contribution)
    off[:, 2, 0, :] = 0.5      # k = 1 at y = 0: h = -0.5 (only the lower corners)
    off[:, 12, H - 1, :] = 0.0  # k = 6 at y = H-1: h = H exactly (no contribution)
    off[:, 14, H - 1, :] = -1.0  # k = 7 at y = H-1: h = H-1 exactly (integer, upper corners outside)
    off[:, 17, :, 3] = 100.0   # k = 8: far outside
    off[:, 9, :, 4] = -50.0    # k = 4: far outside in w
    got, want = _im2col_case(cuda, x, off)
    r = assert_close(got, want, 1e-6, "deform im2col, exact positions")
    parity_log(f"[depthnet] deform im2col exact: rel_max {r:.2e}")
    assert torch.equal(got.double().cpu(), want)


def test_deform_im2col_random(cuda):
    n, C, H, W = 3, 256, 16, 44
    g = torch.Generator().manual_seed(11)
    x = torch.randn(n, C, H, W, generator=g)
    off = 2.5 * torch.randn(n, 18, H, W, generator=g)
    got, want = _im2col_case(cuda, x, off)
    # the fp32 samples are within 1e-6; their S32 storage (hi + lo bf16) adds up to 2^-18 of the value
    r = assert_close(got, want, 1e-5, "deform im2col, random offsets")
    parity_log(f"[depthnet] deform im2col random: rel_max {r:.2e}")


# ------------------------------------------------------------------ 5. whole DepthNet
CASES = {  # name: (cin, mid, ctx, D, cam, B, N, fH, fW)
    "nusc_r50": (512, 512, 128, 112, 27, 1, 6, 16, 44),
    "kitti": (640, 640, 128, 112, 33, 1, 1, 24, 80),
}


def _inputs(case, seed=12):
    cin, _, _, _, cam, B, N, fH, fW = CASES[case]
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B * N, cin, fH, fW, generator=g), torch.randn(B, N, cam, generator=g)


@pytest.mark.parametrize("case", list(CASES))
def test_depthnet_against_fp64(cuda, case):
    cin, mid, ctx, D, cam = CASES[case][:5]
    net = _net(cin, mid, ctx, D, cam, 13, cuda)
    x, mlp = _inputs(case)
    y = net(x.to(cuda), mlp.to(cuda))
    with torch.no_grad():
        want = f64(net)(x.double(), mlp.double())
    rd = assert_close(y[:, :D], want[:, :D], 1e-3, f"DepthNet {case} depth logits")
    rc = assert_close(y[:, D:], want[:, D:], 1e-3, f"DepthNet {case} context")
    parity_log(f"[depthnet] {case}: depth rel_max {rd:.2e}, context rel_max {rc:.2e}")


# ------------------------------------------------------------------ 6. connected: the view transformer from the config
@pytest.mark.parametrize("case", ["nusc_r50", "kitti"])
def test_view_transformer_from_config(cuda, case):
    cin, mid, ctx, D, cam, B, N, fH, fW = CASES[case]
    vt, cams, mlp = config_view_transformer(case, 14, B)
    assert (vt.numC_input, vt.depth_net.mid_channels, vt.cam_channels, vt.D, vt.numC_Trans) == (cin, mid, cam, D, ctx)
    vt = vt.to(cuda)
    g = torch.Generator().manual_seed(15)
    x = torch.randn(B, N, cin, fH, fW, generator=g)
    inp = [x.to(cuda)] + [cams[k].to(cuda) for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    bev, prob = vt(inp + [mlp.to(cuda)])
    assert twin_of(bev) is not None and twin_of(bev).shape == bev.permute(0, 2, 3, 4, 1).shape
    with torch.no_grad():
        out = f64(vt.depth_net)(x.view(B * N, cin, fH, fW).double(), mlp.double())
    check_pooled(vt, cams, out, prob, bev, B, N, f"[depthnet] view transformer {case}", "exact")


# ------------------------------------------------------------------ 7. only library kernels, graph-safe
def test_only_library_kernels_and_cuda_graph(cuda):
    res = run_trace("depthnet", 600)
    assert res["counted"] == res["kernels"] + res["memsets"] and 20 <= res["counted"] <= 40
    assert res["graph_equals_eager"], "CUDA-graph replay differs from the eager forward"


# ------------------------------------------------------------------ 8. bf16 mode
def test_bf16_mode(cuda):
    cin, mid, ctx, D, cam = CASES["nusc_r50"][:5]
    net = _net(cin, mid, ctx, D, cam, 18, cuda)
    x, mlp = _inputs("nusc_r50", seed=19)
    with ops.precision("bf16"):
        y = net(x.to(cuda), mlp.to(cuda))
    with torch.no_grad():
        want = f64(net)(x.double(), mlp.double())
    rd = assert_close(y[:, :D], want[:, :D], 3e-2, "DepthNet bf16 depth logits")
    rc = assert_close(y[:, D:], want[:, D:], 3e-2, "DepthNet bf16 context")
    parity_log(f"[depthnet] bf16 mode: depth rel_max {rd:.2e}, context rel_max {rc:.2e}")


# ------------------------------------------------------------------ 9. shape contract
def test_shape_contract(cuda):
    net = _net(32, 32, 16, 8, 27, 20, cuda)  # mid 32: 8 channels per DCN group
    g = torch.Generator().manual_seed(21)
    x, mlp = torch.randn(2, 32, 6, 9, generator=g), torch.randn(1, 2, 27, generator=g)
    with pytest.raises(RuntimeError, match="mid_channels a multiple of 128"):
        net(x.to(cuda), mlp.to(cuda))
    y = net.cpu()(x, mlp)  # the CPU forward still runs
    assert y.shape == (2, 24, 6, 9)
    big = _net(64, 128, 32, 16, 27, 22, cuda).train()
    with pytest.raises(RuntimeError, match="eval mode"):
        big(torch.randn(2, 64, 6, 9, device=cuda), torch.randn(1, 2, 27, device=cuda))
