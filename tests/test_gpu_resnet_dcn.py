"""ResNetDCN on the library's kernels (image_encoder.py ResNetDCN._bottleneck_cuda): the modulated deformable im2col one
launch at a time against an fp64 restatement of mmcv's sampling, the DCN Bottlenecks, the whole R101-DCN at the nuScenes
R101 size, the chain images -> R101-DCN -> SECONDFPN -> view transformer, the launch count and CUDA-graph replay
(tests/forward_trace.py r101, in a process of its own), the shape contract and the bf16 mode.  The module oracle is
image_encoder.py's torch forward in float64 on the GPU (pinned on the host by tests/test_cpu_resnet_dcn.py)."""
import json
import os

import pytest
import torch

from util import GOLDEN, assert_close, bits, f64, images, parity_log, rel_err, rel_rms, run_trace
from vt_chain import check_pooled
from occformer_b200 import BACKBONES, NECKS, ops, synth
from occformer_b200.common import twin_of
from occformer_b200.image_encoder import SECONDFPN, ModulatedDeformConv2dPack, ResNetDCN

pytestmark = pytest.mark.gpu

KERNEL_TOL = 5e-5
R101 = dict(style="caffe", dcn=dict(type="DCNv2", deform_groups=1, fallback_on_stride=False),
            stage_with_dcn=(False, False, True, True))
FPN = dict(in_channels=[256, 512, 1024, 2048], out_channels=[128, 128, 128, 128], upsample_strides=[0.25, 0.5, 1, 2])
HW = (896, 1600)


def _backbone(seed, dev, **kw):
    net = ResNetDCN(101, **R101).eval()
    net.load_state_dict(synth.make_resnet_dcn_state(seed, **R101, **kw), strict=True)
    return net.to(dev)


def _neck(seed, dev):
    net = SECONDFPN(**FPN).eval()
    net.load_state_dict(synth.make_secondfpn_state(seed=seed, **FPN), strict=True)
    return net.to(dev)


def r101_view_transformer(seed, B):
    """The view transformer of tests/golden/model_cfg_nusc_r101.json (eval mode, on the host) with six nuScenes cameras
    at the config's 896x1600 input size and the synthetic DepthNet state of `seed`, its mlp_input BatchNorm1d running
    statistics matched to those cameras, as vt_chain.config_view_transformer does for the other configs.
    -> (vt, cams, mlp_input)"""
    vt = NECKS.build(json.load(open(os.path.join(GOLDEN, "model_cfg_nusc_r101.json")))["img_view_transformer"])
    dn = vt.depth_net
    sd = synth.make_depthnet_state(dn.in_channels, dn.mid_channels, dn.context_channels, dn.depth_channels,
                                   dn.cam_channels, seed=seed)
    cams = synth.workload_cameras("nusc_r101", B)
    assert tuple(synth.WORKLOADS["nusc_r101"]["input_size"]) == tuple(vt.data_config["input_size"]) == HW
    mlp = vt.get_mlp_input(cams["rots"], cams["trans"], cams["intrins"], cams["post_rots"], cams["post_trans"],
                           cams["bda"])
    sd["bn.running_mean"] = mlp.reshape(-1, dn.cam_channels).mean(0)
    sd["bn.running_var"] = mlp.reshape(-1, dn.cam_channels).var(0, unbiased=False) + 1.0
    dn.load_state_dict(sd, strict=True)
    return vt.eval(), cams, mlp


def ref_modulated_cols(x, off, n, H, W):
    """mmcv's modulated_deformable_im2col_gpu_kernel in fp64: x (n*H*W, C) values, off (n*H*W, >= 27) fp32 -> (n*H*W,
    9*C).  The sample coordinate is formed with the kernel's own fp32 add (an fp32 model has no other), the rest in fp64:
    zero unless h > -1 && w > -1 && h < H && w < W, bilinear with corners outside the map zero, times sigmoid(logit)."""
    C = x.shape[1]
    x = x.double()
    o = off.view(n, H, W, -1)
    b = torch.arange(n, device=x.device).view(n, 1, 1)
    ys = torch.arange(H, device=x.device).view(1, H, 1)
    xs = torch.arange(W, device=x.device).view(1, 1, W)
    out = []
    for k in range(9):
        h = ((ys - 1 + k // 3).float() + o[..., 2 * k]).double()
        w = ((xs - 1 + k % 3).float() + o[..., 2 * k + 1]).double()
        inside = (h > -1) & (w > -1) & (h < H) & (w < W)
        hl, wl = h.floor(), w.floor()
        lh, lw = h - hl, w - wl
        val = 0
        for dy, dx, wt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
            yy, xx = (hl + dy).long(), (wl + dx).long()
            ok = inside & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
            idx = ((b * H + yy.clamp(0, H - 1)) * W + xx.clamp(0, W - 1)).reshape(-1)
            val = val + (wt * ok).reshape(-1, 1) * x[idx]
        out.append(val * torch.sigmoid(o[..., 18 + k].double()).reshape(-1, 1))
    return torch.stack(out, 1).reshape(n * H * W, 9 * C)


# ------------------------------------------------------------------ 1. the modulated im2col, one launch
@pytest.mark.parametrize("n,H,W,C,kind", [(2, 28, 50, 256, "eighths"), (2, 56, 100, 64, "random"),
                                          (3, 5, 7, 512, "random"), (2, 3, 6, 256, "border"), (1, 4, 3, 64, "far"),
                                          (4, 14, 25, 512, "eighths")])
def test_modulated_deform_im2col_against_fp64(cuda, n, H, W, C, kind):
    """offsets on the 1/8-pixel grid (exact bilinear weights), random ones of about 1 px, +-3 px on maps smaller than 8
    (most samples at or over the border), and samples 1e3 px off the map; channels 27..31 of the offset rows hold NaN
    and must not matter"""
    g = torch.Generator().manual_seed(n * 1000 + H * 10 + C)
    rows = n * H * W
    x = ops.to_split(torch.randn(rows, C, generator=g).to(cuda))
    scale = {"eighths": 1.5, "random": 1.0, "border": 3.0, "far": 1e3}[kind]
    off = torch.randn(rows, 32, generator=g) * scale
    if kind == "eighths":
        off = (off * 8).round() / 8
    elif kind == "far":
        off = torch.where(off >= 0, 1e3, -1e3)
    off[:, 18:27] = torch.randn(rows, 9, generator=g) * 2
    off[:, 27:] = float("nan")
    off = off.to(cuda)
    n0 = ops.LAUNCH_COUNT[0]
    cols = ops.modulated_deform_im2col(x, off, n, H, W)
    assert ops.LAUNCH_COUNT[0] - n0 == 1 and cols.shape == (rows, 9 * C)
    want = ref_modulated_cols(ops.from_split(x), off, n, H, W)
    got = ops.from_split(cols)
    if kind == "far":
        assert bool((bits(cols) == 0).all()), "a sample 1e3 px off the map contributed"
    else:
        r = assert_close(got, want, KERNEL_TOL, f"modulated im2col {kind} n{n} {H}x{W} C{C}")
        parity_log(f"[resnet dcn] modulated deform im2col {kind} n{n} {H}x{W} C{C}: rel_max {r:.2e}")
    assert torch.equal(bits(cols), bits(ops.modulated_deform_im2col(x, off, n, H, W)))  # repeat: bit-identical
    if kind == "border":
        o = off.view(n, H, W, 32).cpu()
        ys, xs = torch.arange(H).view(1, H, 1), torch.arange(W).view(1, 1, W)
        outside = sum(float(((ys - 1 + k // 3 + o[..., 2 * k] <= -1) | (ys - 1 + k // 3 + o[..., 2 * k] >= H) |
                             (xs - 1 + k % 3 + o[..., 2 * k + 1] <= -1) |
                             (xs - 1 + k % 3 + o[..., 2 * k + 1] >= W)).double().mean()) for k in range(9)) / 9
        assert 0.2 < outside < 0.9, f"{outside:.0%} of the samples off the map"


def test_modulated_deform_im2col_rejects(cuda):
    x = torch.zeros(2 * 4 * 4, 48, device=cuda)
    with pytest.raises(RuntimeError, match="argument error"):
        ops.modulated_deform_im2col(x, torch.zeros(32, 32, device=cuda), 2, 4, 4)  # C % 32
    x = torch.zeros(32, 64, device=cuda)
    with pytest.raises(RuntimeError, match="argument error"):
        ops.modulated_deform_im2col(x, torch.zeros(32, 18, device=cuda), 2, 4, 4)  # no mask columns


# ------------------------------------------------------------------ 2. DCN Bottlenecks
@pytest.mark.parametrize("block,cin,hw", [(0, 512, (96, 160)), (1, 1024, (48, 80))])
def test_dcn_bottleneck_against_fp64(cuda, block, cin, hw):
    """layer3.0 (caffe: stride-2 conv1, downsample) and layer3.1 (identity shortcut), with bn3 weights around 1 so that
    the DCN branch is as large as the identity path"""
    net = _backbone(40, cuda, bn3_gain=1.0)
    idx = 3 + 4 + block
    x = torch.randn(2, cin, *hw, generator=torch.Generator().manual_seed(41)).abs()
    x_cl = x.permute(0, 2, 3, 1).contiguous().to(cuda).unsqueeze(3)
    p = net.prepared()["blocks"][idx]
    assert p[5] and p[6] is not None
    x_s = ops.to_split(x_cl)
    n0 = ops.LAUNCH_COUNT[0]
    out, out_s = ResNetDCN._bottleneck_cuda(p, x_cl, x_s)
    assert ops.LAUNCH_COUNT[0] - n0 == 6 + (block == 0)  # a plain Bottleneck's 4 (+ downsample) + conv_offset + im2col
    with torch.no_grad():
        want = f64(net, cuda).layer3[block](x.double().to(cuda)).permute(0, 2, 3, 1)
    r = assert_close(out[:, :, :, 0], want, 1e-3, f"DCN Bottleneck layer3.{block}")
    assert torch.equal(bits(out_s), bits(ops.to_split(out)))
    parity_log(f"[resnet dcn] DCN Bottleneck layer3.{block}: rel_max {r:.2e}")


# ------------------------------------------------------------------ 3. the whole backbone at full size
def test_r101_dcn_full_size_against_fp64(cuda):
    net = _backbone(42, cuda)
    x = images(6, *HW, seed=43)
    outs = net(x.to(cuda))
    ref = f64(net, cuda)
    offs = []
    hooks = [m.conv_offset.register_forward_hook(lambda m, i, o: offs.append(o.float().cpu()))
             for m in ref.modules() if isinstance(m, ModulatedDeformConv2dPack)]
    with torch.no_grad():
        want = ref._forward_torch(x.double().to(cuda))
    for h in hooks:
        h.remove()
    assert len(outs) == 4 and len(offs) == 26
    for i, (o, wnt) in enumerate(zip(outs, want)):
        assert o.shape == wnt.shape and o.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(bits(twin_of(o)), bits(ops.to_split(o.permute(0, 2, 3, 1).contiguous())))
        r = assert_close(o, wnt, 1e-3, f"R101-DCN stage {i}")
        pos = float((wnt > 0).double().mean())
        assert 0.05 < pos < 0.95, f"stage {i}: {pos:.1%} positive activations -- a vacuous comparison"
        parity_log(f"[resnet dcn] R101-DCN (6, 3, 896, 1600) stage {i}: rel_max {r:.2e}, {pos:.0%} positive")
    outside, frac, mid = 0.0, 0.0, 0.0
    for o in offs:
        _, _, h, w = o.shape
        ys, xs = torch.arange(h).view(1, h, 1), torch.arange(w).view(1, 1, w)
        for k in range(9):
            sy, sx = ys - 1 + k // 3 + o[:, 2 * k], xs - 1 + k % 3 + o[:, 2 * k + 1]
            outside += float(((sy <= -1) | (sx <= -1) | (sy >= h) | (sx >= w)).double().mean())
            frac += float(((sy != sy.round()) & (sx != sx.round())).double().mean())
        m = torch.sigmoid(o[:, 18:27])
        mid += float(((m > 0.1) & (m < 0.9)).double().mean())
    outside, frac, mid = outside / (9 * len(offs)), frac / (9 * len(offs)), mid / len(offs)
    parity_log(f"[resnet dcn] R101-DCN samples off the map {outside:.2%}, fractional {frac:.0%}, masks in (0.1, 0.9) "
               f"{mid:.0%}")
    assert outside > 0.005 and frac > 0.9 and mid > 0.5, (outside, frac, mid)


# ------------------------------------------------------------------ 4. connected: images -> view transformer
def test_images_to_view_transformer(cuda):
    """images -> ResNetDCN (built from the unmodified R101 config with the class opted in) -> SECONDFPN -> the view
    transformer of the unmodified R101 config at 896x1600, against the same chain in float64 (oracle.port lift /
    pooling), gated as test_gpu_image_encoder.py::test_images_to_view_transformer"""
    cfg = json.load(open(os.path.join(GOLDEN, "image_encoder_cfg_nusc_r101.json")))
    backbone = BACKBONES.build(dict(cfg["img_backbone"], type=ResNetDCN)).eval()
    neck = NECKS.build(cfg["img_neck"]).eval()
    backbone.load_state_dict(synth.make_resnet_dcn_state(44, **R101), strict=True)
    neck.load_state_dict(synth.make_secondfpn_state(seed=45, **FPN), strict=True)
    B, N = 1, 6
    vt, cams, mlp = r101_view_transformer(46, B)
    backbone, neck, vt = backbone.to(cuda), neck.to(cuda), vt.to(cuda)
    imgs = images(B * N, *HW, seed=47)

    feat = neck(backbone(imgs.to(cuda)))[0]
    _, C, H, W = feat.shape
    assert (C, H, W) == (512, 56, 100)
    x = feat.view(B, N, C, H, W)
    inp = [x] + [cams[k].to(cuda) for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    bev, prob = vt(inp + [mlp.to(cuda)])

    with torch.no_grad():
        stages = f64(backbone, cuda)._forward_torch(imgs.double().to(cuda))
        feat64 = f64(neck, cuda)._forward_torch(list(stages))[0]
        out = f64(vt.depth_net, cuda)._forward_torch(feat64, mlp.double().to(cuda)).cpu()
    del stages
    check_pooled(vt, cams, out, prob, bev, B, N, "[resnet dcn] R101 images -> view transformer", "terms")


# ------------------------------------------------------------------ 5. only library kernels, graph-safe
def test_only_library_kernels_and_cuda_graph(cuda):
    res = run_trace("r101", 1500)
    assert res["memsets"] == 0
    # stem im2col + GEMM + max-pool, 33 Bottlenecks x (3 convs + split) + 4 downsamples, 26 DCNs x (conv_offset +
    # modulated im2col), SECONDFPN: 2 space_to_depth + 3 convs + GEMM + depth_to_space
    assert res["counted"] == res["kernels"] == 3 + 33 * 4 + 4 + 26 * 2 + 7 == 198
    assert res["graph_equals_eager"], "CUDA-graph replay differs from the eager forward"


# ------------------------------------------------------------------ 6. shape contract, bf16 mode
def test_shape_contract(cuda):
    net = ResNetDCN(50, **R101).eval().to(cuda)
    x = images(1, 100, 128, seed=48)
    with pytest.raises(RuntimeError, match="ResNetDCN's CUDA forward needs H and W multiples of 32"):
        net(x.to(cuda))
    assert net.cpu()(x)[3].shape == (1, 2048, 4, 4)  # the CPU forward still runs
    net = net.to(cuda).train()
    with pytest.raises(RuntimeError, match="eval mode"):
        net(images(1, 64, 64).to(cuda))


def test_bf16_mode(cuda):
    backbone, neck = _backbone(49, cuda), _neck(50, cuda)
    x = images(6, *HW, seed=51)
    with ops.precision("bf16"):
        y = neck(list(backbone(x.to(cuda))))[0]
    with torch.no_grad():
        want = f64(neck, cuda)._forward_torch(list(f64(backbone, cuda)._forward_torch(x.double().to(cuda))))[0]
    # single-pass bf16 operands (~3e-3 per contraction) through 104 stacked convs, 26 deformable samplings whose
    # positions come from bf16 contractions, and the FPN; a mode without a reference twin: bounded by its max and rms
    # error (2.9e-2 / 2.1e-2 measured on H100)
    r, q = rel_err(y, want), rel_rms(y, want)
    parity_log(f"[resnet dcn] bf16 mode: rel_max {r:.2e}, rel_rms {q:.2e}")
    assert r <= 6e-2 and q <= 4e-2, f"R101-DCN bf16: rel_max {r:.2e}, rel_rms {q:.2e}"
