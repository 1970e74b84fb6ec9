"""DepthNet of the LSS view transformer -- SURVEY.md 8(f)3: the caller in front of the lift-splat hot path.

    DepthNet / ASPP / Mlp / SELayer      projects/mmdet3d_plugin/occformer/image2bev/ViewTransformerLSSBEVDepth.py:330-504
    BasicBlock                           mmdet 2.14.0 mmdet/models/backbones/resnet.py (conv1, bn1, conv2, bn2)
    DCN (mmcv DeformConv2dPack)          mmcv-full 1.4.0 mmcv/ops/deform_conv.py (weight, conv_offset.{weight,bias})

The module tree has the reference's exact ``state_dict`` keys and shapes, so that a reference checkpoint's
``img_view_transformer.depth_net.*`` entries load with ``strict=True``.  Inference only: BatchNorm uses its running
statistics (eval mode), as in the reference's test path.

On CUDA tensors ``forward`` runs on this package's sm_90a kernels (``_forward_cuda``, about 30 launches, no host
synchronisation, CUDA-graph capturable): every convolution -- reduce_conv, the BasicBlocks, the ASPP branches and
projection, conv_offset, the DCN's four group contractions, the 1x1 heads -- is the fp32-faithful implicit-GEMM conv
(occ_conv_bf16x3 / occ_conv_slice_bf16x3) with the eval BatchNorms folded in once per weight set (``_prepare``); the
camera-aware SE gates, their application, the ASPP pooling branch and the deformable im2col are small kernels of their
own (csrc/depthnet_ops.cu).  A CUDA input outside that path's shape contract raises RuntimeError; there is no fallback.
On CPU tensors ``forward`` is the plain torch restatement ``_forward_torch`` (the oracle of the GPU tests, pinned to the
reference class by tests/golden/depthnet_small.npz).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .common import PreparedModule, fold_bn


class BasicBlock(nn.Module):
    """mmdet ResNet BasicBlock with stride 1, no downsample (DepthNet.depth_conv[0:3])."""

    def __init__(self, inplanes, planes):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        return self.relu(out + x)


class _ASPPModule(nn.Module):
    def __init__(self, inplanes, planes, kernel_size, padding, dilation):
        super().__init__()
        self.atrous_conv = nn.Conv2d(inplanes, planes, kernel_size, stride=1, padding=padding, dilation=dilation, bias=False)
        self.bn = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU()

    def forward(self, x):
        return self.relu(self.bn(self.atrous_conv(x)))


class ASPP(nn.Module):
    """ViewTransformerLSSBEVDepth.py:349-414 (dropout 0.5 is the identity in eval)."""

    def __init__(self, inplanes, mid_channels=256):
        super().__init__()
        d = [1, 6, 12, 18]
        self.aspp1 = _ASPPModule(inplanes, mid_channels, 1, 0, d[0])
        self.aspp2 = _ASPPModule(inplanes, mid_channels, 3, d[1], d[1])
        self.aspp3 = _ASPPModule(inplanes, mid_channels, 3, d[2], d[2])
        self.aspp4 = _ASPPModule(inplanes, mid_channels, 3, d[3], d[3])
        self.global_avg_pool = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), nn.Conv2d(inplanes, mid_channels, 1, bias=False),
                                             nn.BatchNorm2d(mid_channels), nn.ReLU())
        self.conv1 = nn.Conv2d(5 * mid_channels, mid_channels, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(mid_channels)
        self.relu = nn.ReLU()
        self.dropout = nn.Dropout(0.5)

    def forward(self, x):
        x5 = F.interpolate(self.global_avg_pool(x), size=x.shape[2:], mode="bilinear", align_corners=True)
        y = torch.cat((self.aspp1(x), self.aspp2(x), self.aspp3(x), self.aspp4(x), x5), dim=1)
        return self.dropout(self.relu(self.bn1(self.conv1(y))))


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features, out_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = nn.ReLU()
        self.drop1 = nn.Dropout(0.0)
        self.fc2 = nn.Linear(hidden_features, out_features)
        self.drop2 = nn.Dropout(0.0)

    def forward(self, x):
        return self.drop2(self.fc2(self.drop1(self.act(self.fc1(x)))))


class SELayer(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv_reduce = nn.Conv2d(channels, channels, 1, bias=True)
        self.act1 = nn.ReLU()
        self.conv_expand = nn.Conv2d(channels, channels, 1, bias=True)
        self.gate = nn.Sigmoid()

    def forward(self, x, x_se):
        return x * self.gate(self.conv_expand(self.act1(self.conv_reduce(x_se))))


def deform_columns(x, off):
    """The sampling columns of a 3x3, stride 1, padding 1 deformable conv with one deformable group (mmcv DeformConv2d /
    ModulatedDeformConv2d): x (B, C, H, W), off (B, >= 18, H, W) whose channel 2k / 2k+1 is the (dy, dx) offset of
    kernel point k = ky*3 + kx -> (B, C, 9, H, W), point k sampled at (y - 1 + ky + dy, x - 1 + kx + dx), bilinear with
    zeros outside the map (``grid_sample``)."""
    B, C, H, W = x.shape
    ys = torch.arange(H, device=x.device, dtype=x.dtype).view(1, H, 1)
    xs = torch.arange(W, device=x.device, dtype=x.dtype).view(1, 1, W)
    cols = []
    for k in range(9):
        py = ys + (k // 3 - 1) + off[:, 2 * k]
        px = xs + (k % 3 - 1) + off[:, 2 * k + 1]
        grid = torch.stack((2.0 * px / max(W - 1, 1) - 1.0, 2.0 * py / max(H - 1, 1) - 1.0), dim=-1)
        cols.append(F.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=True))
    return torch.stack(cols, dim=2)


class DCN(nn.Module):
    """mmcv ``DeformConv2dPack`` (DCNv1): 3x3, stride 1, padding 1, ``groups`` weight groups, one deformable group.
    Parameters: ``weight`` (out, in/groups, 3, 3) without bias and ``conv_offset`` = Conv2d(in, 18, 3, padding 1) whose
    output channel 2k / 2k+1 is the (dy, dx) offset of kernel point k.  Forward: bilinear sampling with zeros outside the
    map (``grid_sample``), then the grouped contraction."""

    def __init__(self, in_channels, out_channels, kernel_size=3, padding=1, groups=4, **_):
        super().__init__()
        assert kernel_size == 3 and padding == 1
        self.groups = groups
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, 3, 3))
        nn.init.kaiming_uniform_(self.weight, nonlinearity="relu")
        self.conv_offset = nn.Conv2d(in_channels, 18, 3, stride=1, padding=1, bias=True)
        nn.init.zeros_(self.conv_offset.weight)
        nn.init.zeros_(self.conv_offset.bias)

    def forward(self, x):
        B, C, H, W = x.shape
        col = deform_columns(x, self.conv_offset(x))  # (B, C, 9, H, W)
        g = self.groups
        col = col.view(B, g, C // g, 9, H, W)
        w = self.weight.view(g, -1, C // g, 9)  # (g, out/g, in/g, 9)
        return torch.einsum("bgckhw,gock->bgohw", col, w).reshape(B, -1, H, W)


class DepthNet(PreparedModule):
    """ViewTransformerLSSBEVDepth.py:450-504: camera-aware depth / context heads.  forward(x (B*N, Cin, fH, fW),
    mlp_input (B, N, cam_channels)) -> (B*N, D + C_ctx, fH, fW) = depth logits | context features."""

    def __init__(self, in_channels, mid_channels, context_channels, depth_channels, cam_channels=27):
        super().__init__()
        self.in_channels, self.mid_channels, self.context_channels = in_channels, mid_channels, context_channels
        self.depth_channels, self.cam_channels = depth_channels, cam_channels
        self.reduce_conv = nn.Sequential(nn.Conv2d(in_channels, mid_channels, 3, stride=1, padding=1),
                                         nn.BatchNorm2d(mid_channels), nn.ReLU(inplace=True))
        self.context_conv = nn.Conv2d(mid_channels, context_channels, 1)
        self.bn = nn.BatchNorm1d(cam_channels)
        self.depth_mlp = Mlp(cam_channels, mid_channels, mid_channels)
        self.depth_se = SELayer(mid_channels)
        self.context_mlp = Mlp(cam_channels, mid_channels, mid_channels)
        self.context_se = SELayer(mid_channels)
        self.depth_conv = nn.Sequential(BasicBlock(mid_channels, mid_channels), BasicBlock(mid_channels, mid_channels),
                                        BasicBlock(mid_channels, mid_channels), ASPP(mid_channels, mid_channels),
                                        DCN(mid_channels, mid_channels, 3, padding=1, groups=4),
                                        nn.Conv2d(mid_channels, depth_channels, 1))

    def forward(self, x, mlp_input):
        """x (B*N, Cin, fH, fW), mlp_input (B, N, cam_channels) -> (B*N, D + C_ctx, fH, fW)."""
        if x.is_cuda:
            return self._forward_cuda(x, mlp_input)
        return self._forward_torch(x, mlp_input)

    # ------------------------------------------------------------------ parameters of the CUDA forward
    @torch.no_grad()
    def _folded(self):
        """Eval-mode BatchNorms folded into the layer before them (common.fold_bn; natural layouts, on the parameters'
        device).  Also the BatchNorm1d of mlp_input folded into both fc1's, conv_offset padded to 32 output channels and
        the DCN weight as `groups` tap-major matrices (Cout/groups, 9 * Cin/groups), column k * Cin/groups + c."""
        def plain(layer):
            return layer.weight.detach().float().contiguous(), layer.bias.detach().float().contiguous()

        F_ = {}
        F_["reduce"] = fold_bn(self.reduce_conv[0].weight, self.reduce_conv[0].bias, self.reduce_conv[1])
        F_["ctx"] = plain(self.context_conv)
        s = self.bn.weight.double() / torch.sqrt(self.bn.running_var.double() + self.bn.eps)
        t = self.bn.bias.double() - self.bn.running_mean.double() * s  # bn(m) = s * m + t
        gates = []
        for mlp, se in ((self.depth_mlp, self.depth_se), (self.context_mlp, self.context_se)):
            w1 = mlp.fc1.weight.double()
            gates.append(((w1 * s.view(1, -1)).float(), (mlp.fc1.bias.double() + w1 @ t).float(),
                          *plain(mlp.fc2), se.conv_reduce.weight.detach().float()[:, :, 0, 0], se.conv_reduce.bias.detach().float(),
                          se.conv_expand.weight.detach().float()[:, :, 0, 0], se.conv_expand.bias.detach().float()))
        F_["gates"] = tuple(torch.stack([a, b]).contiguous() for a, b in zip(*gates))  # (2, ...) depth | context
        F_["blocks"] = [fold_bn(blk.conv1.weight, None, blk.bn1) + fold_bn(blk.conv2.weight, None, blk.bn2)
                        for blk in self.depth_conv[:3]]
        aspp = self.depth_conv[3]
        F_["aspp"] = [fold_bn(m.atrous_conv.weight, None, m.bn)
                      for m in (aspp.aspp1, aspp.aspp2, aspp.aspp3, aspp.aspp4)]
        gw, gb = fold_bn(aspp.global_avg_pool[1].weight, None, aspp.global_avg_pool[2])
        F_["gap"] = (gw[:, :, 0, 0].contiguous(), gb)
        F_["aspp_c1"] = fold_bn(aspp.conv1.weight, None, aspp.bn1)
        dcn = self.depth_conv[4]
        ow, ob = plain(dcn.conv_offset)
        F_["offset"] = (torch.cat([ow, ow.new_zeros(32 - ow.shape[0], *ow.shape[1:])]).contiguous(),
                        torch.cat([ob, ob.new_zeros(32 - ob.shape[0])]).contiguous())
        g = dcn.groups
        w = dcn.weight.detach().float()  # (Cout, Cin/g, 3, 3)
        Og, Cg = w.shape[0] // g, w.shape[1]
        F_["dcn"] = w.view(g, Og, Cg, 9).permute(0, 1, 3, 2).reshape(g, Og, 9 * Cg).contiguous()
        F_["depth"] = plain(self.depth_conv[5])
        return F_

    @torch.no_grad()
    def _prepare(self):
        """The folded parameters in the kernels' layouts: conv weights repacked tap-major in S32, the gate weights
        K-major (in, out), the DCN group matrices in S32."""
        F_ = self._folded()
        P = {}
        P["reduce"] = (ops.repack_conv_weight(F_["reduce"][0])[0], F_["reduce"][1])
        P["ctx"] = (ops.repack_conv_weight(F_["ctx"][0])[0], F_["ctx"][1])
        w1, b1, w2, b2, wr, br, we, be = F_["gates"]
        kmaj = lambda w: w.transpose(1, 2).contiguous()  # noqa: E731
        P["gates"] = (kmaj(w1), b1, kmaj(w2), b2, kmaj(wr), br, kmaj(we), be)
        P["blocks"] = [(ops.repack_conv_weight(a)[0], ab, ops.repack_conv_weight(b)[0], bb) for a, ab, b, bb in F_["blocks"]]
        P["aspp"] = [(ops.repack_conv_weight(w)[0], b) for w, b in F_["aspp"]]
        P["gap"] = F_["gap"]
        P["aspp_c1"] = (ops.repack_conv_weight(F_["aspp_c1"][0])[0], F_["aspp_c1"][1])
        P["offset"] = (ops.repack_conv_weight(F_["offset"][0])[0], F_["offset"][1])
        P["dcn"] = [ops.split_weight(m) for m in F_["dcn"]]
        P["depth"] = (ops.repack_conv_weight(F_["depth"][0])[0], F_["depth"][1])
        return P

    def _check_cuda_contract(self, x, mlp_input):
        n, cin = x.shape[0], x.shape[1]
        need = []
        if x.dim() != 4 or cin != self.in_channels:
            need.append(f"x of shape (B*N, {self.in_channels}, fH, fW)")
        if cin % 32:
            need.append("in_channels % 32 == 0 (whole 32-channel chunks of the conv operand)")
        if self.mid_channels % 128 or self.mid_channels > 1024:
            need.append(f"mid_channels a multiple of 128 up to 1024 (each of the DCN's {self.depth_conv[4].groups} groups "
                        "is whole 32-channel chunks)")
        if self.depth_conv[4].groups != 4:
            need.append("DCN groups == 4")
        if self.depth_channels % 4 or self.context_channels % 4:
            need.append("depth_channels % 4 == 0 and context_channels % 4 == 0 (16-byte column slices of the output)")
        if self.cam_channels > 256 or mlp_input is None or mlp_input.numel() != n * self.cam_channels:
            need.append("mlp_input with B*N x cam_channels elements, cam_channels <= 256")
        if n > 65535:
            need.append("B*N <= 65535")
        if self.training:
            need.append("eval mode (the CUDA forward applies the BatchNorms' running statistics; call .eval())")
        if need:
            raise RuntimeError(f"occformer_b200: DepthNet's CUDA forward needs {'; '.join(need)} -- got "
                               f"x {tuple(x.shape)}, DepthNet({self.in_channels}, {self.mid_channels}, "
                               f"{self.context_channels}, {self.depth_channels}, cam_channels={self.cam_channels})")

    @torch.no_grad()
    def _forward_cuda(self, x, mlp_input):
        self._check_cuda_contract(x, mlp_input)
        P = self.prepared()
        n, Cin, H, W = x.shape
        HW, rows = H * W, x.shape[0] * H * W
        C, D, Cc = self.mid_channels, self.depth_channels, self.context_channels
        k3, k1 = (3, 3, 1), (1, 1, 1)

        def img(t, c):  # (rows, c) channel-last rows -> the conv's (images, H, W, 1, c) view
            return t.view(n, H, W, 1, c)

        x_s = ops.split_nchw(x.float()).view(n, HW, Cin)  # -> channel-last S32 (no transpose for a channels_last map)
        gates = ops.depthnet_cam_gates(mlp_input.reshape(n, -1).float().contiguous(), *P["gates"])
        xr = ops.conv(img(x_s, Cin), P["reduce"][0], k3, bias=P["reduce"][1], act=1).view(rows, C)
        xd, xd_s, xc_s = ops.se_apply(xr, gates, n, HW)
        # (rows, D + C_ctx): depth logits | context, transposed to the reference's layout at the end
        out_cl = torch.empty((rows, D + Cc), dtype=torch.float32, device=x.device)
        ops.conv_into(img(xc_s, C), P["ctx"][0], k1, out_cl, D, bias=P["ctx"][1])
        cur, cur_s = xd, xd_s
        for w1, b1, w2, b2 in P["blocks"]:  # relu(bn2(conv2(relu(bn1(conv1(x))))) + x)
            t_s = ops.conv(img(cur_s, C), w1, k3, bias=b1, act=1, split_out=True)
            cur = ops.conv(t_s, w2, k3, bias=b2, residual=cur, act=1).view(rows, C)
            cur_s = ops.to_split(cur)
        cat = torch.empty((rows, 5 * C), dtype=torch.float32, device=x.device)  # S32 concat of the five ASPP branches
        for i, ((w, b), d) in enumerate(zip(P["aspp"], (1, 6, 12, 18))):
            ops.conv_into(img(cur_s, C), w, k1 if i == 0 else k3, cat, i * C, dil=d if i else 1, bias=b, act=1,
                          split_out=True)
        ops.depthnet_gap_branch(cur, *P["gap"], cat, n, HW, 4 * C)
        a_s = ops.conv(img(cat, 5 * C), P["aspp_c1"][0], k1, bias=P["aspp_c1"][1], act=1, split_out=True)
        off = ops.conv(a_s, P["offset"][0], k3, bias=P["offset"][1]).view(rows, 32)
        g = len(P["dcn"])
        cols = ops.deform_im2col(a_s, off, n, H, W, g)
        dcn_s = torch.empty((rows, C), dtype=torch.float32, device=x.device)
        for i, wg in enumerate(P["dcn"]):
            ops.conv_into(img(cols[i], 9 * C // g), wg, k1, dcn_s, i * C // g, split_out=True)
        ops.conv_into(img(dcn_s, C), P["depth"][0], k1, out_cl, 0, bias=P["depth"][1])
        return ops.transpose_sq(out_cl.view(n, HW, D + Cc), n, HW, D + Cc).view(n, D + Cc, H, W)

    # ------------------------------------------------------------------ the torch restatement (CPU path, test oracle)
    def _forward_torch(self, x, mlp_input):
        mlp_input = self.bn(mlp_input.reshape(-1, mlp_input.shape[-1]))
        x = self.reduce_conv(x)
        context = self.context_conv(self.context_se(x, self.context_mlp(mlp_input)[..., None, None]))
        depth = self.depth_conv(self.depth_se(x, self.depth_mlp(mlp_input)[..., None, None]))
        return torch.cat([depth, context], dim=1)
