"""Deterministic synthetic inputs for the hot path (SURVEY.md 8(d)): nuScenes-like fixed camera
constants, seeded CPU generation.  Shared by tests/ and bench.py so that the oracle and the CUDA
path always see identical tensors.  No dataset, no checkpoint: everything is synthetic."""
import math

import torch

GRIDS = {
    # name: (xbound, ybound, zbound)            -> X x Y x Z
    "pr1": ([-20.0, 20.0, 0.8], [-20.0, 20.0, 0.8], [-2.0, 4.4, 0.8]),          # 50 x 50 x 8
    "nusc_ref": ([-51.2, 51.2, 0.8], [-51.2, 51.2, 0.8], [-5.0, 3.0, 0.5]),     # 128 x 128 x 16
    "nusc_200": ([-40.0, 40.0, 0.4], [-40.0, 40.0, 0.4], [-1.0, 5.4, 0.4]),     # 200 x 200 x 16
    "kitti": ([0.0, 51.2, 0.4], [-25.6, 25.6, 0.4], [-2.0, 4.4, 0.4]),          # 128 x 128 x 16 (occformer_kitti.py:22-46)
}
DBOUND = [2.0, 58.0, 0.5]


def grid_config(name):
    xb, yb, zb = GRIDS[name]
    return {"xbound": xb, "ybound": yb, "zbound": zb, "dbound": DBOUND}


def _yaw(deg):
    a = math.radians(deg)
    c, s = math.cos(a), math.sin(a)
    return torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


CAM2EGO_AXES = torch.tensor([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])


# the workloads of BASELINE.json `configs` (shapes: SURVEY.md section 8 legend): cameras, input, lift grid, output grid, classes
WORKLOADS = {
    "nusc_200": dict(name="nusc_r50_6cam_256x704_to_200x200x16", cams=6, input_size=(256, 704), grid="nusc_200",
                     occ=[200, 200, 16], pc=[-40.0, -40.0, -1.0, 40.0, 40.0, 5.4], classes=17, head="Mask2FormerNuscOccHead"),
    "nusc_ref": dict(name="nusc_r50_6cam_256x704_to_128x128x16_occ256x256x32", cams=6, input_size=(256, 704), grid="nusc_ref",
                     occ=[256, 256, 32], pc=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], classes=17, head="Mask2FormerNuscOccHead"),
    "kitti": dict(name="semantickitti_1cam_384x1280_to_128x128x16_occ256x256x32", cams=1, input_size=(384, 1280), grid="kitti",
                  occ=[256, 256, 32], pc=[0.0, -25.6, -2.0, 51.2, 25.6, 4.4], classes=20, head="Mask2FormerOccHead"),
    "nusc_r101": dict(name="nusc_r101_6cam_896x1600_to_200x200x16", cams=6, input_size=(896, 1600), grid="nusc_200",
                      occ=[200, 200, 16], pc=[-40.0, -40.0, -1.0, 40.0, 40.0, 5.4], classes=17, head="Mask2FormerNuscOccHead"),
    # occformer_nusc_panoptic_r50_256x704.py: the reference grid, 150 queries, thing classes barrier .. truck
    "nusc_panoptic": dict(name="nusc_panoptic_r50_6cam_256x704_to_128x128x16_occ256x256x32", cams=6, input_size=(256, 704),
                          grid="nusc_ref", occ=[256, 256, 32], pc=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], classes=17,
                          head="Mask2FormerNuscPanopticOccHead", queries=150, thing_indices=list(range(1, 11))),
}


def workload_cameras(wl, B=1):
    w = WORKLOADS[wl]
    return kitti_camera(B, w["input_size"]) if wl == "kitti" else nusc_cameras(B, w["cams"], w["input_size"])


def nusc_cameras(B=1, N=6, input_size=(256, 704)):
    """Six cameras, yaw {+55,0,-55,+110,180,-110} deg; intrinsics of a 1600x900 nuScenes camera;
    post_rot/post_tran of the reference's test-time resize+crop (loading_nusc_imgs.py:85-93)."""
    yaws = [55.0, 0.0, -55.0, 110.0, 180.0, -110.0][:N]
    H, W = input_size
    resize = W / 1600.0
    crop_h = int(900 * resize) - H
    rots = torch.stack([_yaw(y) @ CAM2EGO_AXES for y in yaws])
    trans = torch.tensor([[1.5 * math.cos(math.radians(y)), 1.5 * math.sin(math.radians(y)), 1.5] for y in yaws])
    K = torch.tensor([[1266.4, 0.0, 816.3], [0.0, 1266.4, 491.5], [0.0, 0.0, 1.0]])
    intrins = K.expand(N, 3, 3)
    post_rots = torch.diag(torch.tensor([resize, resize, 1.0])).expand(N, 3, 3)
    post_trans = torch.tensor([0.0, -float(crop_h), 0.0]).expand(N, 3)
    bda = torch.eye(3)

    def rep(t):
        return t.unsqueeze(0).repeat(B, *([1] * t.dim())).contiguous()

    return dict(rots=rep(rots), trans=rep(trans), intrins=rep(intrins), post_rots=rep(post_rots),
                post_trans=rep(post_trans), bda=rep(bda))


def kitti_camera(B=1, input_size=(384, 1280)):
    """SemanticKITTI-like single left camera (BASELINE.json configs[1]): 4x4 P2 intrinsics with the shift column
    (semantic_kitti_lss_dataset.py:62-64 hands a 4x4 matrix over), camera -> LiDAR axes, 4x4 homogeneous bda."""
    H, W = input_size
    resize = W / 1226.0
    rots = (_yaw(0.0) @ CAM2EGO_AXES).view(1, 1, 3, 3).repeat(B, 1, 1, 1)
    trans = torch.tensor([0.27, 0.0, -0.08]).view(1, 1, 3).repeat(B, 1, 1)
    K = torch.eye(4)
    K[:3, :4] = torch.tensor([[707.09, 0.0, 604.08, 45.76], [0.0, 707.09, 180.51, -0.35], [0.0, 0.0, 1.0, 0.005]])
    post_rots = torch.diag(torch.tensor([resize, resize, 1.0])).view(1, 1, 3, 3).repeat(B, 1, 1, 1)
    post_trans = torch.tensor([0.0, -float(int(370 * resize) - H), 0.0]).view(1, 1, 3).repeat(B, 1, 1)
    return dict(rots=rots.contiguous(), trans=trans.contiguous(), intrins=K.view(1, 1, 4, 4).repeat(B, 1, 1, 1).contiguous(),
                post_rots=post_rots.contiguous(), post_trans=post_trans.contiguous(),
                bda=torch.eye(4).view(1, 4, 4).repeat(B, 1, 1).contiguous())


def pr1_camera(B=1):
    """One front camera, 128x128, fx=fy=100, cx=cy=64 (BASELINE.json configs[0])."""
    rots = (_yaw(0.0) @ CAM2EGO_AXES).view(1, 1, 3, 3).repeat(B, 1, 1, 1)
    trans = torch.tensor([1.5, 0.0, 1.5]).view(1, 1, 3).repeat(B, 1, 1)
    K = torch.tensor([[100.0, 0.0, 64.0], [0.0, 100.0, 64.0], [0.0, 0.0, 1.0]])
    return dict(rots=rots, trans=trans, intrins=K.view(1, 1, 3, 3).repeat(B, 1, 1, 1),
                post_rots=torch.eye(3).view(1, 1, 3, 3).repeat(B, 1, 1, 1),
                post_trans=torch.zeros(B, 1, 3), bda=torch.eye(3).view(1, 3, 3).repeat(B, 1, 1))


def lift_inputs(B, N, D, fH, fW, C, seed=0):
    """Post-DepthNet tensors: depth logits ~ 3*N(0,1) (B*N,D,fH,fW), context ~ N(0,1) (B*N,C,fH,fW)."""
    g = torch.Generator().manual_seed(seed)
    depth_digit = 3.0 * torch.randn(B * N, D, fH, fW, generator=g)
    img_feat = torch.randn(B * N, C, fH, fW, generator=g)
    return depth_digit, img_feat


def encoder_input(B, C, X, Y, Z, seed=0):
    g = torch.Generator().manual_seed(seed)
    return 0.5 * torch.randn(B, C, X, Y, Z, generator=g)


def head_inputs(B, E, sizes, seed=0):
    """voxel_feats list, high -> low resolution: [mask_features, level2, level1, level0]."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, E, *s, generator=g) * (0.5 if i == 0 else 1.0) for i, s in enumerate(sizes)]


def lidar_points(n, pc_range, seed=0):
    g = torch.Generator().manual_seed(seed)
    lo = torch.tensor(pc_range[:3])
    hi = torch.tensor(pc_range[3:])
    pts = lo + (hi - lo) * (torch.rand(n, 3, generator=g) * 1.1 - 0.05)  # a few out of range
    return torch.cat([pts, torch.zeros(n, 2)], dim=1)


# =============================================================================
# deterministic synthetic weights (same keys / shapes as the reference modules, SURVEY.md Appendix B)
# =============================================================================
def rel_position_index(ws=7):
    """WindowMSA.relative_position_index (window_attention.py:57-61, 109-113): double_step_seq + flip."""
    seq1 = torch.arange(0, (2 * ws - 1) * ws, 2 * ws - 1)
    seq2 = torch.arange(0, ws, 1)
    c = (seq1[:, None] + seq2[None, :]).reshape(1, -1)
    return (c + c.T).flip(1).contiguous()



def _randn(g, *shape, std=1.0):
    return torch.randn(*shape, generator=g) * std


def make_block_state(cin, c, stride, g, prefix=""):
    """state_dict of one DualpathTransformerBlock (SURVEY Appendix B), seeded generator ``g``.
    Zero-initialised reference params are perturbed so that they matter (SURVEY 8(d))."""
    sd = {}
    p = prefix

    def norm(name, n):
        sd[p + name + "weight"] = 1 + 0.1 * _randn(g, n)
        sd[p + name + "bias"] = 0.1 * _randn(g, n)

    def lin(name, o, i):
        sd[p + name + "weight"] = _randn(g, o, i, std=i ** -0.5)
        sd[p + name + "bias"] = 0.1 * _randn(g, o)

    if stride > 1:
        sd[p + "downsample.0.weight"] = _randn(g, c, cin, 1, 1, 1, std=cin ** -0.5)
        norm("downsample.1.", c)
    sd[p + "input_conv.0.weight"] = _randn(g, c, cin, 3, 3, 3, std=(27 * cin) ** -0.5)
    norm("input_conv.1.", c)
    be = "bev_encoder."
    norm(be + "norm1.", c)
    sd[p + be + "attn.w_msa.relative_position_bias_table"] = _randn(g, 169, c // 32, std=0.5)
    sd[p + be + "attn.w_msa.relative_position_index"] = rel_position_index(7)
    lin(be + "attn.w_msa.qkv.", 3 * c, c)
    lin(be + "attn.w_msa.proj.", c, c)
    norm(be + "norm2.", c)
    lin(be + "ffn.layers.0.0.", c, c)
    lin(be + "ffn.layers.1.", c, c)
    ch = c // 4
    sd[p + "aspp.input_conv.0.weight"] = _randn(g, ch, c, 1, 1, std=c ** -0.5)
    norm("aspp.input_conv.1.", ch)
    sd[p + "aspp.aspp.aspp1.atrous_conv.weight"] = _randn(g, ch, ch, 1, 1, std=ch ** -0.5)
    norm("aspp.aspp.aspp1.bn.", ch)
    for i in (2, 3, 4):
        sd[p + f"aspp.aspp.aspp{i}.atrous_conv.weight"] = _randn(g, ch, ch, 3, 3, std=(9 * ch) ** -0.5)
        norm(f"aspp.aspp.aspp{i}.bn.", ch)
    sd[p + "aspp.aspp.global_avg_pool.1.weight"] = _randn(g, ch, ch, 1, 1, std=ch ** -0.5)
    norm("aspp.aspp.global_avg_pool.2.", ch)
    sd[p + "aspp.aspp.conv1.weight"] = _randn(g, ch, 5 * ch, 1, 1, std=(5 * ch) ** -0.5)
    norm("aspp.aspp.bn1.", ch)
    sd[p + "aspp.output_conv.0.weight"] = _randn(g, c, ch, 1, 1, std=ch ** -0.5)
    norm("aspp.output_conv.1.", c)
    sd[p + "combine_coeff.weight"] = _randn(g, 1, c, 1, 1, 1, std=c ** -0.5)
    sd[p + "combine_coeff.bias"] = 0.1 * _randn(g, 1)
    return sd


def make_encoder_state(in_channels, block_inplanes, block_numbers, block_strides, seed=0, prefix=""):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    cin = in_channels
    for s, (c, nb, st) in enumerate(zip(block_inplanes, block_numbers, block_strides)):
        for b in range(nb):
            sd.update(make_block_state(cin, c, st if b == 0 else 1, g, f"{prefix}layers.{s}.{b}."))
            cin = c
    return sd


def make_head_state(E=192, Q=100, K=17, num_layers=9, num_levels=3, ffn=None, seed=0, prefix=""):
    """state_dict of Mask2FormerNuscOccHead (inference params; SURVEY Appendix B)."""
    g = torch.Generator().manual_seed(seed)
    ffn = ffn or 8 * E
    sd = {}
    p = prefix

    def norm(name):
        sd[p + name + "weight"] = 1 + 0.1 * _randn(g, E)
        sd[p + name + "bias"] = 0.1 * _randn(g, E)

    def lin(name, o, i, wname="weight", bname="bias"):
        sd[p + name + wname] = _randn(g, o, i, std=i ** -0.5)
        sd[p + name + bname] = 0.1 * _randn(g, o)

    sd[p + "query_embed.weight"] = _randn(g, Q, E)
    sd[p + "query_feat.weight"] = _randn(g, Q, E)
    sd[p + "level_embed.weight"] = _randn(g, num_levels, E)
    lin("cls_embed.", K + 1, E)
    for i in (0, 2, 4):
        lin(f"mask_embed.{i}.", E, E)
    for l in range(num_layers):
        lp = f"transformer_decoder.layers.{l}."
        for a in (0, 1):
            lin(lp + f"attentions.{a}.attn.", 3 * E, E, "in_proj_weight", "in_proj_bias")
            lin(lp + f"attentions.{a}.attn.out_proj.", E, E)
        lin(lp + "ffns.0.layers.0.0.", ffn, E)
        lin(lp + "ffns.0.layers.1.", E, ffn)
        for n in (0, 1, 2):
            norm(lp + f"norms.{n}.")
    norm("transformer_decoder.post_norm.")
    return sd


def make_neck_state(in_channels, E, num_layers, num_heads, num_levels=3, num_points=4, ffn=None, seed=0):
    """Deterministic weights with the reference's state_dict keys.  Unlike the reference's init (zero sampling-offset
    and attention-weight matrices), every matrix is non-trivial so that a parity test moves the sampling points."""
    g = torch.Generator().manual_seed(seed)
    ffn = ffn or 4 * E
    sd = {}

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    def gn(name, n):
        sd[name + "weight"] = 1.0 + 0.1 * rn(n)
        sd[name + "bias"] = 0.1 * rn(n)

    nin = len(in_channels)
    for i in range(num_levels):
        cin = in_channels[nin - i - 1]
        sd[f"input_convs.{i}.conv.weight"] = rn(E, cin, 1, 1, 1, std=cin ** -0.5)
        sd[f"input_convs.{i}.conv.bias"] = 0.1 * rn(E)
        gn(f"input_convs.{i}.gn.", E)
    for l in range(num_layers):
        p = f"encoder.layers.{l}."
        n_off = num_heads * num_levels * num_points
        sd[p + "attentions.0.sampling_offsets.weight"] = rn(3 * n_off, E, std=0.5 * E ** -0.5)
        sd[p + "attentions.0.sampling_offsets.bias"] = rn(3 * n_off, std=1.0)
        sd[p + "attentions.0.attention_weights.weight"] = rn(n_off, E, std=E ** -0.5)
        sd[p + "attentions.0.attention_weights.bias"] = 0.1 * rn(n_off)
        for nm in ("value_proj", "output_proj"):
            sd[p + f"attentions.0.{nm}.weight"] = rn(E, E, std=E ** -0.5)
            sd[p + f"attentions.0.{nm}.bias"] = 0.1 * rn(E)
        sd[p + "ffns.0.layers.0.0.weight"] = rn(ffn, E, std=E ** -0.5)
        sd[p + "ffns.0.layers.0.0.bias"] = 0.1 * rn(ffn)
        sd[p + "ffns.0.layers.1.weight"] = rn(E, ffn, std=ffn ** -0.5)
        sd[p + "ffns.0.layers.1.bias"] = 0.1 * rn(E)
        gn(p + "norms.0.", E)
        gn(p + "norms.1.", E)
    sd["level_encoding.weight"] = rn(num_levels, E)
    for i in range(nin - num_levels):
        sd[f"lateral_convs.{i}.conv.weight"] = rn(E, in_channels[i], 1, 1, 1, std=in_channels[i] ** -0.5)
        gn(f"lateral_convs.{i}.gn.", E)
        sd[f"output_convs.{i}.conv.weight"] = rn(E, E, 3, 3, 3, std=(27 * E) ** -0.5)
        gn(f"output_convs.{i}.gn.", E)
    sd["mask_feature.weight"] = rn(E, E, 1, 1, 1, std=E ** -0.5)
    sd["mask_feature.bias"] = 0.1 * rn(E)
    return sd


def make_depthnet_state(cin, mid, ctx, D, cam=27, seed=0):
    """state_dict of DepthNet(cin, mid, ctx, D, cam) (depthnet.py, the reference's keys): seeded weights and non-trivial
    BatchNorm statistics (running mean ~ 0.1 N(0,1), running var in [0.5, 1.5]).  conv_offset is scaled so that the DCN
    offsets are a few pixels: some sampling points fall outside the map."""
    from .depthnet import DepthNet
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in DepthNet(cin, mid, ctx, D, cam_channels=cam).state_dict().items():
        if k.endswith("num_batches_tracked"):
            sd[k] = v.clone()
        elif k.endswith("running_mean"):
            sd[k] = 0.1 * _randn(g, *v.shape)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(*v.shape, generator=g)
        elif v.dim() == 1 and not k.endswith("bias"):  # BatchNorm weight
            sd[k] = 1 + 0.1 * _randn(g, *v.shape)
        elif k == "depth_conv.4.conv_offset.weight":
            sd[k] = _randn(g, *v.shape, std=1.5 * v[0].numel() ** -0.5)
        elif k == "depth_conv.4.conv_offset.bias":
            sd[k] = _randn(g, *v.shape, std=1.5)
        elif k.endswith("bias"):
            sd[k] = 0.1 * _randn(g, *v.shape)
        else:  # conv / linear weight (out, in, ...): unit gain over the fan-in
            sd[k] = _randn(g, *v.shape, std=v[0].numel() ** -0.5)
    return sd


@torch.no_grad()
def _calibrate_batchnorms(net, inputs, g, jitter=0.05, floor=0.01):
    """Running statistics of every BatchNorm2d of the CPU module ``net`` from one float64 forward on ``inputs``: each
    BatchNorm gets the batch mean / variance of its own input (variance floored at ``floor`` (1 %) of its channel mean, so
    that no channel that happens to be dead at this size is amplified 300x at another), perturbed slightly (mean + jitter *
    std * N(0,1), var * (1 + jitter * U(-1,1))).  The statistics are set before each BatchNorm runs, so every layer is
    calibrated on already calibrated activations.  -> the float32 state_dict"""
    import torch.nn as nn
    net = net.double().eval()

    def pre(bn, args):
        x = args[0]
        mean, var = x.mean((0, 2, 3)), x.var((0, 2, 3), unbiased=False)
        var = var + floor * var.mean()
        bn.running_mean.copy_(mean + jitter * var.sqrt() * _randn(g, *mean.shape).double())
        bn.running_var.copy_(var * (1 + jitter * (2 * torch.rand(*var.shape, generator=g).double() - 1)))

    hooks = [m.register_forward_pre_hook(pre) for m in net.modules() if isinstance(m, nn.BatchNorm2d)]
    try:
        net(*inputs)
    finally:
        for h in hooks:
            h.remove()
    return {k: (v.float() if v.is_floating_point() else v).clone() for k, v in net.state_dict().items()}


def _he_state(net, g):
    """He-initialised conv weights (std sqrt(2 / fan_in); a ConvTranspose2d's fan-in is its in_channels), BatchNorm
    weight 1 + 0.1 N(0,1), BatchNorm / conv bias 0.1 N(0,1); running statistics left for calibration"""
    import torch.nn as nn
    sd = {}
    for name, m in net.named_modules():
        p = name + "." if name else ""
        if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
            fan_in = m.weight[0].numel() if isinstance(m, nn.Conv2d) else m.weight.shape[0]
            sd[p + "weight"] = _randn(g, *m.weight.shape, std=(2.0 / fan_in) ** 0.5)
            if m.bias is not None:
                sd[p + "bias"] = 0.1 * _randn(g, *m.bias.shape)
        elif isinstance(m, nn.BatchNorm2d):
            sd[p + "weight"] = 1 + 0.1 * _randn(g, m.num_features)
            sd[p + "bias"] = 0.1 * _randn(g, m.num_features)
    net.load_state_dict(sd, strict=False)
    return net


def make_resnet_state(seed=0, calib_shape=(4, 3, 64, 96), **resnet_kwargs):
    """state_dict of image_encoder.ResNet(depth=50, **resnet_kwargs) (mmdet's keys = torchvision resnet50's without fc.*):
    He-initialised convs, BatchNorm affine 1 + 0.1 N / 0.1 N, and running statistics calibrated on a seeded fp64 forward
    of N(0,1) images of calib_shape (then perturbed slightly), so that the 16 stacked blocks neither vanish nor blow up
    on images of that kind at any size.  No BatchNorm weight is zero.

    The last BatchNorm of each residual branch (bn3) has weight 0.25 (1 + 0.1 N): the branch is smaller than the identity
    path, as in trained ResNets.  With bn3 weights around 1 the random stack is chaotic: a relative perturbation of 1e-5
    of every conv weight grows to 3e-3 at layer4 (fp64 on the host), so no fp32 implementation, cuDNN's included, could
    be compared with another at the 1e-3 gate."""
    from .image_encoder import ResNet
    g = torch.Generator().manual_seed(seed)
    net = _he_state(ResNet(depth=50, **resnet_kwargs), g)
    with torch.no_grad():
        for name, m in net.named_modules():
            if name.endswith(".bn3"):
                m.weight.mul_(0.25)
    return _calibrate_batchnorms(net, [_randn(g, *calib_shape).double()], g)


def make_resnet_dcn_state(seed=0, depth=101, calib_shape=(1, 3, 224, 416), bn3_gain=0.05, **resnet_kwargs):
    """state_dict of image_encoder.ResNetDCN(depth, **resnet_kwargs), made as make_resnet_state makes ResNet's (He convs,
    bn3 weight bn3_gain * (1 + 0.1 N), BatchNorm statistics calibrated on a seeded fp64 forward of N(0,1) images of
    calib_shape), with each DCNv2's weight He-initialised and its conv_offset He-initialised with zero bias: on the
    calibrated, ReLU'd input of the DCN, offsets of about 1 px (std 1.07 at the R101 config; fractional positions
    everywhere, about 3 % of the samples off the map) and mask logits of about N(0, 1) (std 1.07).

    bn3_gain is smaller than make_resnet_state's 0.25 because R101 stacks 23 blocks in layer3, and a DCN block also
    passes its input on through the sampling positions.  Measured in fp64 on the host at the R101 config (style 'caffe',
    DCN in layer3 / layer4) as the growth of a relative perturbation of 1e-5 of every conv / DCN / BatchNorm weight,
    layer1 .. layer4 on (1, 3, 448, 800) images: 4.1e-5, 5.0e-5, 9.2e-5, 1.8e-4 at bn3_gain 0.05; 1.1e-3 / 1.7e-3 at
    layer3 / layer4 with 0.1 and 0.18 / 0.43 with 0.25 (chaotic: no two fp32 implementations could meet the 1e-3 gate).
    Without the DCNs, caffe-style R101 at 0.25 reaches 7.1e-4 at layer4 ((1, 3, 224, 416) images)."""
    from .image_encoder import ModulatedDeformConv2dPack, ResNetDCN
    g = torch.Generator().manual_seed(seed)
    net = _he_state(ResNetDCN(depth=depth, **resnet_kwargs), g)
    with torch.no_grad():
        for name, m in net.named_modules():
            if name.endswith(".bn3"):
                m.weight.mul_(bn3_gain)
            elif isinstance(m, ModulatedDeformConv2dPack):
                m.weight.copy_(_randn(g, *m.weight.shape, std=(2.0 / m.weight[0].numel()) ** 0.5))
                m.conv_offset.bias.zero_()
    return _calibrate_batchnorms(net, [_randn(g, *calib_shape).double()], g)


def make_secondfpn_state(in_channels, out_channels, upsample_strides, seed=0, out_hw=(4, 8), n=2, **fpn_kwargs):
    """state_dict of image_encoder.SECONDFPN(in_channels, out_channels, upsample_strides, **fpn_kwargs) (the reference's
    deblocks.{i}.{0,1}.* keys): He-initialised (de)convs, BatchNorm affine 1 + 0.1 N / 0.1 N, running statistics
    calibrated on seeded non-negative (post-ReLU-like) levels |N(0,1)| whose sizes map to out_hw."""
    from .image_encoder import SECONDFPN
    g = torch.Generator().manual_seed(seed)
    net = _he_state(SECONDFPN(in_channels, out_channels, upsample_strides, **fpn_kwargs), g)
    levels = [_randn(g, n, c, int(out_hw[0] / s), int(out_hw[1] / s)).abs() for c, s in zip(in_channels, upsample_strides)]
    return _calibrate_batchnorms(net, [[t.double() for t in levels]], g)


def make_efficientnet_state(arch="b7", seed=0, calib_shape=(1, 3, 384, 1280), linear_bn_gain=0.25, floor=16.0, **kwargs):
    """state_dict of efficientnet.CustomEfficientNet(arch, **kwargs) (the reference's keys): He-initialised convs (the
    SE convs too, with bias 0.1 N), BatchNorm affine 1 + 0.1 N / 0.1 N, and running statistics calibrated on a seeded fp64
    forward of N(0,1) images of calib_shape (then perturbed slightly), so that the stacked blocks neither vanish nor blow
    up on images of that size.

    Three things keep B7's 55 random blocks from being chaotic (measured in fp64 on the host as the growth of a 1e-5
    relative perturbation of every conv / BatchNorm weight; at 1e-3 or more no two fp32 implementations could be compared
    at the 1e-3 gate):
    - each block's last BatchNorm (linear_conv.bn, before the residual add) has weight linear_bn_gain * (1 + 0.1 N), as
      ResNet's bn3 in make_resnet_state: the branch is smaller than the identity path, as in trained networks;
    - the calibrated variances are floored at ``floor`` = 16x the layer's mean channel variance (make_resnet_state:
      1 %), so that no near-constant channel is lifted 10x; every BatchNorm then scales its channels down about 4x, and
      the Swish after it works near its linear part;
    - the calibration images have the KITTI size.  Calibrated at 96x320, layers.5 sees 3x10 maps on which most 5x5
      depthwise taps fall into the padding; at 384x1280 its interior pixels then have a larger variance than calibrated.
    Measured at (1, 3, 384, 1280), calibrated there: the perturbation reaches 2.1e-4 at layers.6 (floor 4x: 5.2e-4; 1 %
    floor and calibration at 96x320: 0.43 already at 192x640).
    About half of every stage's activations are positive."""
    from .efficientnet import CustomEfficientNet
    g = torch.Generator().manual_seed(seed)
    net = _he_state(CustomEfficientNet(arch=arch, **kwargs), g)
    with torch.no_grad():
        for name, m in net.named_modules():
            if name.endswith("linear_conv.bn"):
                m.weight.mul_(linear_bn_gain)
    return _calibrate_batchnorms(net, [_randn(g, *calib_shape).double()], g, floor=floor)


def make_detector_state(cfg, seed=0, cams=None):
    """state_dict of detector.OccupancyFormer(**cfg) for a reference config's ``model`` dict, keys prefixed and in the
    order a reference checkpoint lists them: each submodule's synthetic state above, seeded from seed .. seed + 6, plus
    the view transformer's geometry parameters (dx, bx, nx, frustum) as the module computes them.  With ``cams`` (a
    camera dict as workload_cameras makes) DepthNet's mlp_input BatchNorm1d gets the statistics of those cameras' MLP
    input (variance + 1), as a trained model's would; otherwise make_depthnet_state's."""
    from .detector import OccupancyFormer
    from .image_encoder import ResNet, ResNetDCN
    cfg = {k: v for k, v in cfg.items() if k != "type"}
    det = OccupancyFormer(**cfg)
    subs = {}
    h = det.pts_bbox_head
    subs["pts_bbox_head"] = make_head_state(h.decoder_embed_dims, h.num_queries, h.num_classes,
                                            h.num_transformer_decoder_layers, h.num_transformer_feat_level,
                                            ffn=h.ffn_channels, seed=seed)
    bb = {k: v for k, v in cfg["img_backbone"].items() if k not in ("type", "pretrained", "init_cfg")}
    if isinstance(det.img_backbone, ResNetDCN):
        subs["img_backbone"] = make_resnet_dcn_state(seed + 1, **bb)
    elif isinstance(det.img_backbone, ResNet):
        bb.pop("depth")
        subs["img_backbone"] = make_resnet_state(seed + 1, **bb)
    else:
        subs["img_backbone"] = make_efficientnet_state(seed=seed + 1, **bb)
    neck = {k: v for k, v in cfg["img_neck"].items() if k != "type"}
    # calibrated on the level sizes the image-encoder tests use (KITTI: stride-32 levels of 192 x 640 images)
    subs["img_neck"] = make_secondfpn_state(seed=seed + 2, **neck, **({} if isinstance(det.img_backbone, ResNet)
                                                                     else dict(out_hw=(6, 20))))
    vt = det.img_view_transformer
    dn = vt.depth_net
    sd = make_depthnet_state(dn.in_channels, dn.mid_channels, dn.context_channels, dn.depth_channels, dn.cam_channels,
                             seed=seed + 3)
    if cams is not None:
        mlp = vt.get_mlp_input(cams["rots"], cams["trans"], cams["intrins"], cams["post_rots"], cams["post_trans"],
                               cams["bda"]).reshape(-1, dn.cam_channels)
        sd["bn.running_mean"] = mlp.mean(0)
        sd["bn.running_var"] = mlp.var(0, unbiased=False) + 1.0
    vsd = {k: v for k, v in vt.state_dict().items() if not k.startswith("depth_net.")}
    vsd.update({"depth_net." + k: v for k, v in sd.items()})
    subs["img_view_transformer"] = vsd
    e = cfg["img_bev_encoder_backbone"]
    subs["img_bev_encoder_backbone"] = make_encoder_state(e["in_channels"], e["block_inplanes"], e["block_numbers"],
                                                          e["block_strides"], seed=seed + 5)
    n = det.img_bev_encoder_neck
    ffn = n.state_dict()["encoder.layers.0.ffns.0.layers.0.0.weight"].shape[0]
    subs["img_bev_encoder_neck"] = make_neck_state(n.in_channels, n.embed_dims, len(n.encoder.layers), n.num_heads,
                                                   n.num_encoder_levels, n.num_points, ffn, seed=seed + 6)
    order = [k for k in det.state_dict()]
    flat = {f"{m}.{k}": v for m, s in subs.items() for k, v in s.items()}
    return {k: flat[k] for k in order if k in flat} | {k: v for k, v in flat.items() if k not in order}
