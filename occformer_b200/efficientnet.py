"""Image encoder of the SemanticKITTI model: the EfficientNet backbone in front of SECONDFPN and DepthNet.

    CustomEfficientNet / InvertedResidual / model_scaling   P/occformer/backbones/efficientnet.py:112-229,231-519
    mmcv 1.4.0 Conv2dAdaptivePadding, Swish, ConvModule; mmdet 2.14.0 SELayer, make_divisible (restated below)
    config       projects/configs/occformer_kitti/occformer_kitti.py:66-80 (img_backbone, arch 'b7')

``CustomEfficientNet`` takes the reference's constructor kwargs and builds its exact ``state_dict`` keys (including its
rule of not building the layers after ``max(out_indices)``), so a reference checkpoint's ``img_backbone.*`` entries load
with ``strict=True``.  The 'b0'..'b8' archs are supported.  Inference only: BatchNorm uses its running statistics.

On CUDA tensors ``forward`` runs on this package's sm_90a kernels (``_forward_cuda``, no host synchronisation, CUDA-graph
capturable).  Per InvertedResidual block: the expand 1x1 conv is an fp32-faithful GEMM with Swish in its epilogue; the
depthwise conv, its BatchNorm and Swish are one kernel that also writes the squeeze-and-excitation partial sums; one
kernel per image computes the SE gate, one applies it and writes the linear conv's operand; the linear 1x1 conv is a GEMM
with the residual in its epilogue.  Every channel count is zero-padded to whole 32-channel chunks inside this path (zero
weights, biases and BatchNorm entries), so pad channels are exactly 0 throughout.  A CUDA input outside the path's shape
contract raises RuntimeError; there is no cuDNN fallback.  On CPU tensors ``forward`` is the plain torch restatement
``_forward_torch`` (the oracle of the GPU tests), adaptive padding included.

Stage outputs are handed on as the ResNet's are (image_encoder.py): an fp32 NCHW view of channel-last memory with the
reference's channel count, carrying its S32 twin (common.attach_twin); the twin of a stage whose width is not a
multiple of 32 is zero-padded to whole chunks (SECONDFPN takes such twins).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .common import PreparedModule, attach_twin, batchnorm, fold_bn, round32
from .registry import BACKBONES


def make_divisible(value, divisor, min_value=None, min_ratio=0.9):
    """mmdet 2.14 make_divisible: the nearest multiple of divisor (at least min_value, default divisor), one divisor more
    if rounding lost more than 1 - min_ratio of value"""
    min_value = divisor if min_value is None else min_value
    v = max(min_value, int(value + divisor / 2) // divisor * divisor)
    return v + divisor if v < min_ratio * value else v


def adaptive_pad(size, k, stride, dilation=1):
    """mmcv Conv2dAdaptivePadding along one axis ("same" padding of TF): -> (before, after) with total
    max((ceil(size / stride) - 1) * stride + (k - 1) * dilation + 1 - size, 0), the smaller half before"""
    pad = max((-(-size // stride) - 1) * stride + (k - 1) * dilation + 1 - size, 0)
    return pad // 2, pad - pad // 2


class Swish(nn.Module):
    """mmcv Swish: x * sigmoid(x)"""

    def forward(self, x):
        return x * torch.sigmoid(x)


class Conv2dAdaptivePadding(nn.Conv2d):
    """mmcv Conv2dAdaptivePadding: built without padding; forward pads the input by adaptive_pad (right / bottom get the
    odd pixel) and convolves"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride, 0, dilation, groups, bias)

    def forward(self, x):
        (kh, kw), (sh, sw), (dh, dw) = self.weight.shape[-2:], self.stride, self.dilation
        top, bottom = adaptive_pad(x.shape[-2], kh, sh, dh)
        left, right = adaptive_pad(x.shape[-1], kw, sw, dw)
        if top or bottom or left or right:
            x = F.pad(x, [left, right, top, bottom])
        return F.conv2d(x, self.weight, self.bias, self.stride, 0, self.dilation, self.groups)


class ConvBN(nn.Module):
    """mmcv ConvModule(conv_cfg=Conv2dAdaptivePadding, norm_cfg=BN, act_cfg=Swish | None): conv (no bias) -> bn ->
    [Swish]; keys conv.weight, bn.*"""

    def __init__(self, cin, cout, k, stride=1, groups=1, norm_cfg=None, act=True):
        super().__init__()
        self.conv = Conv2dAdaptivePadding(cin, cout, k, stride, groups=groups, bias=False)
        self.bn = batchnorm(norm_cfg, cout, 1e-5)
        self.activate = Swish() if act else None

    def forward(self, x):
        x = self.bn(self.conv(x))
        return self.activate(x) if self.activate is not None else x


class _ConvAct(nn.Module):
    """mmcv ConvModule without norm: conv with bias -> act; keys conv.weight, conv.bias"""

    def __init__(self, cin, cout, act):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 1)
        self.activate = act

    def forward(self, x):
        return self.activate(self.conv(x))


class SELayer(nn.Module):
    """mmdet 2.14 SELayer(channels, ratio, act_cfg=(Swish, Sigmoid)): x * sigmoid(conv2(swish(conv1(mean_hw(x)))))"""

    def __init__(self, channels, squeeze):
        super().__init__()
        self.global_avgpool = nn.AdaptiveAvgPool2d(1)
        self.conv1 = _ConvAct(channels, squeeze, Swish())
        self.conv2 = _ConvAct(squeeze, channels, nn.Sigmoid())

    def forward(self, x):
        return x * self.conv2(self.conv1(self.global_avgpool(x)))


class InvertedResidual(nn.Module):
    """efficientnet.py:112-229 with SE, in eval: [expand_conv] -> depthwise_conv -> se -> linear_conv (+ x when stride 1
    and cin == cout; DropPath is the identity in eval)"""

    def __init__(self, cin, cout, mid, k, stride, squeeze, norm_cfg):
        super().__init__()
        self.with_expand_conv = mid != cin
        self.with_res_shortcut = stride == 1 and cin == cout
        self.kernel_size, self.stride = k, stride
        if self.with_expand_conv:
            self.expand_conv = ConvBN(cin, mid, 1, norm_cfg=norm_cfg)
        self.depthwise_conv = ConvBN(mid, mid, k, stride, groups=mid, norm_cfg=norm_cfg)
        self.se = SELayer(mid, squeeze)
        self.linear_conv = ConvBN(mid, cout, 1, norm_cfg=norm_cfg, act=False)

    def forward(self, x):
        out = self.expand_conv(x) if self.with_expand_conv else x
        out = self.linear_conv(self.se(self.depthwise_conv(out)))
        return x + out if self.with_res_shortcut else out


# EfficientNet-B0 (Tan & Le, 2019, table 1) as the reference's layer_settings['b']: per layer, blocks of (kernel,
# out_channels, se_ratio, stride, expand_ratio); the first layer is the stem conv, the last the 1x1 head conv
_B0 = [[(3, 32, 0, 2, 0)],
       [(3, 16, 4, 1, 1)],
       [(3, 24, 4, 2, 6), (3, 24, 4, 1, 6)],
       [(5, 40, 4, 2, 6), (5, 40, 4, 1, 6)],
       [(3, 80, 4, 2, 6), (3, 80, 4, 1, 6), (3, 80, 4, 1, 6), (5, 112, 4, 1, 6), (5, 112, 4, 1, 6), (5, 112, 4, 1, 6)],
       [(5, 192, 4, 2, 6), (5, 192, 4, 1, 6), (5, 192, 4, 1, 6), (5, 192, 4, 1, 6), (3, 320, 4, 1, 6)],
       [(1, 1280, 0, 1, 0)]]
_ARCHS = {"b0": (1.0, 1.0), "b1": (1.0, 1.1), "b2": (1.1, 1.2), "b3": (1.2, 1.4), "b4": (1.4, 1.8), "b5": (1.6, 2.2),
          "b6": (1.8, 2.6), "b7": (2.0, 3.1), "b8": (2.2, 3.6)}  # (width, depth) multipliers
_EDGE_ARCHS = ("es", "em", "el")


def scaled_layers(width, depth):
    """the reference's model_scaling on the B0 table: every width times `width`, rounded by make_divisible(., 8); every
    run of consecutive blocks of one width lengthened to ceil(depth * length) blocks (repeating its last block) or cut to
    it; a run whose first block has stride 1 joins the layer before it, except the first run.  -> list of layers, each a
    list of (kernel, out_channels, se_ratio, stride, expand_ratio)"""
    scaled = [[(k, make_divisible(c * width, 8), se, s, e) for k, c, se, s, e in layer] for layer in _B0]
    runs = []
    for layer in scaled[1:-1]:
        start = 0
        for i in range(1, len(layer) + 1):
            if i == len(layer) or layer[i][1] != layer[i - 1][1]:
                runs.append(layer[start:i])
                start = i
    layers = [scaled[0]]
    for i, run in enumerate(runs):
        n = int(math.ceil(depth * len(run)))
        run = run[:n] + [run[-1]] * (n - len(run))
        if run[0][3] == 1 and i != 0:
            layers[-1] = layers[-1] + run
        else:
            layers.append(run)
    return layers + [scaled[-1]]


def _pad(t, *shape):
    """t zero-padded at the end of each dimension to shape"""
    out = t.new_zeros(shape)
    out[tuple(slice(0, s) for s in t.shape)] = t
    return out.contiguous()


@BACKBONES.register_module()
class CustomEfficientNet(PreparedModule):
    """efficientnet.py:274-519 for the 'b' archs: forward(x (n, 3, H, W)) -> tuple of the layers in ``out_indices``
    (layer 0 = stem at stride 2, layers 1..5 the InvertedResidual stages at strides 2, 4, 8, 16, 32, layer 6 the 1x1 head
    conv).  The training-only kwargs (drop_path_rate, with_cp, frozen_stages, norm_eval) and init_cfg are accepted and
    ignored; options this implementation does not have raise NotImplementedError naming the kwarg."""

    def __init__(self, arch="b0", drop_path_rate=0.0, out_indices=(6,), frozen_stages=0,
                 conv_cfg=dict(type="Conv2dAdaptivePadding"), norm_cfg=dict(type="BN", eps=1e-3),
                 act_cfg=dict(type="Swish"), norm_eval=False, with_cp=False, init_cfg=None):
        super().__init__()
        if arch in _EDGE_ARCHS:
            raise NotImplementedError(f"occformer_b200.CustomEfficientNet: arch={arch!r} is not supported (the EdgeTPU "
                                      "archs; 'b0'..'b8' are)")
        if arch not in _ARCHS:
            raise ValueError(f"occformer_b200.CustomEfficientNet: arch={arch!r} is not one of {sorted(_ARCHS)}")
        if dict(conv_cfg or {}).get("type") != "Conv2dAdaptivePadding":
            raise NotImplementedError(f"occformer_b200.CustomEfficientNet: conv_cfg={conv_cfg!r} is not supported "
                                      "(Conv2dAdaptivePadding only)")
        if dict(act_cfg or {}).get("type") != "Swish":
            raise NotImplementedError(f"occformer_b200.CustomEfficientNet: act_cfg={act_cfg!r} is not supported "
                                      "(Swish only)")
        batchnorm(norm_cfg, 1, 1e-5)  # NotImplementedError naming norm_cfg for a non-BatchNorm norm
        if any(i not in range(7) for i in out_indices):
            raise ValueError(f"the item in out_indices must in range(0, 7). But received {tuple(out_indices)}")
        if frozen_stages not in range(8):
            raise ValueError(f"frozen_stages must be in range(0, 8). But received {frozen_stages}")
        self.arch, self.out_indices = arch, tuple(out_indices)
        self.layer_setting = scaled_layers(*_ARCHS[arch])
        stem = self.layer_setting[0][0]
        cin = make_divisible(stem[1], 8)
        self.layers = nn.ModuleList([ConvBN(3, cin, stem[0], stem[3], norm_cfg=norm_cfg)])
        for i, layer in enumerate(self.layer_setting[1:-1]):
            if i > max(self.out_indices) - 1:  # the reference builds no layer after the last output
                break
            blocks = []
            for k, cout, se_ratio, stride, expand in layer:
                mid = int(cin * expand)
                cout = make_divisible(cout, 8)
                blocks.append(InvertedResidual(cin, cout, mid, k, stride, int(mid / (expand * se_ratio)), norm_cfg))
                cin = cout
            self.layers.append(nn.Sequential(*blocks))
        if len(self.layers) < max(self.out_indices) + 1:
            head = self.layer_setting[-1][0]
            self.layers.append(ConvBN(cin, head[1], head[0], head[3], norm_cfg=norm_cfg))

    def forward(self, x):
        if x.is_cuda:
            return self._forward_cuda(x)
        return self._forward_torch(x)

    # ------------------------------------------------------------------ parameters of the CUDA forward
    @torch.no_grad()
    def _prepare(self):
        """The folded parameters in the kernels' layouts, every channel count padded to a multiple of 32 with zeros:
        "stem" (S32 (C0p, 32) in the im2col's (ky, kx, c) column order, bias), "blocks" one dict per InvertedResidual
        (expand / linear S32 (out, in) + bias, depthwise tap-major (k*k, C) + bias, SE K-major w1T (C, S), b1, w2T
        (S, C), b2), "head" (S32 (Cout, Cin), bias) of layers.6 when built.  Each block also records whether its output
        is needed in S32 (the next op is a GEMM, or it ends a stage in out_indices)."""
        def fold(m):
            return fold_bn(m.conv.weight, None, m.bn)

        def gemm_w(w, b):  # 1x1 conv (Cout, Cin, 1, 1) -> S32 (Coutp, Cinp), bias (Coutp)
            co, ci = w.shape[:2]
            return ops.split_weight(_pad(w[:, :, 0, 0], round32(co), round32(ci))), _pad(b, round32(co))

        w, b = fold(self.layers[0])
        c0, k = w.shape[0], w.shape[-1]
        stem = ops.split_weight(_pad(w.permute(0, 2, 3, 1).reshape(c0, 3 * k * k), round32(c0), 32))
        P = {"stem": (stem, _pad(b, round32(c0))), "blocks": [], "head": None}
        stage_ends = {}
        for li, layer in enumerate(self.layers[1:], start=1):
            if not isinstance(layer, nn.Sequential):
                P["head"] = gemm_w(*fold(layer))
                continue
            for blk in layer:
                mid, kk = blk.depthwise_conv.conv.weight.shape[0], blk.kernel_size
                midp = round32(mid)
                wd, bd = fold(blk.depthwise_conv)
                w1, w2 = blk.se.conv1.conv.weight[:, :, 0, 0].float(), blk.se.conv2.conv.weight[:, :, 0, 0].float()
                sq = w1.shape[0]
                se = (_pad(w1.t(), midp, sq), blk.se.conv1.conv.bias.float().contiguous(), _pad(w2.t(), sq, midp),
                      _pad(blk.se.conv2.conv.bias.float(), midp))
                P["blocks"].append(dict(
                    k=kk, stride=blk.stride, res=blk.with_res_shortcut,
                    expand=gemm_w(*fold(blk.expand_conv)) if blk.with_expand_conv else None,
                    dw=(_pad(wd.view(mid, kk * kk).t(), kk * kk, midp), _pad(bd, midp)), se=se,
                    linear=gemm_w(*fold(blk.linear_conv))))
            stage_ends[len(P["blocks"]) - 1] = li
        blocks = P["blocks"]
        for i, p in enumerate(blocks):
            next_is_gemm = blocks[i + 1]["expand"] is not None if i + 1 < len(blocks) else P["head"] is not None
            p["stage"] = stage_ends.get(i)
            p["split"] = next_is_gemm or p["stage"] in self.out_indices
        return P

    def _check_cuda_contract(self, x):
        need = []
        if x.dim() != 4 or x.shape[1] != 3:
            need.append("x of shape (n, 3, H, W)")
        elif x.shape[2] % 32 or x.shape[3] % 32:
            need.append("H and W multiples of 32 (every stage size exact)")
        if x.dim() == 4 and x.shape[0] > 65535:
            need.append("n <= 65535")
        if self.training:
            need.append("eval mode (the CUDA forward applies the BatchNorms' running statistics; call .eval())")
        if need:
            raise RuntimeError(f"occformer_b200: CustomEfficientNet's CUDA forward needs {'; '.join(need)} -- got x "
                               f"{tuple(x.shape)}")

    def _stage(self, cur, cur_s, n, h, w, li):
        """fp32 rows (n*h*w, Cp) + S32 twin -> the NCHW view with the reference's channel count of layer li"""
        C = self._channels(li)
        return attach_twin(cur.view(n, h, w, -1)[..., :C].permute(0, 3, 1, 2), cur_s.view(n, h, w, -1))

    def _channels(self, li):
        layer = self.layers[li]
        last = layer[-1].linear_conv if isinstance(layer, nn.Sequential) else layer
        return last.bn.num_features

    @torch.no_grad()
    def _forward_cuda(self, x):
        self._check_cuda_contract(x)
        P = self.prepared()
        n, _, H, W = x.shape
        stem = self.layers[0].conv
        k, s = stem.weight.shape[-1], stem.stride[0]
        h, w = -(-H // s), -(-W // s)
        cols = ops.im2col3(x.float().contiguous(), k, s, adaptive_pad(H, k, s)[0], adaptive_pad(W, k, s)[0], h, w, 32)
        cur = ops.gemm(cols, P["stem"][0], bias=P["stem"][1], act=3)  # (n*h*w, C0p) fp32
        cur_s = None
        outs = []
        if 0 in self.out_indices:
            cur_s = ops.to_split(cur)
            outs.append(self._stage(cur, cur_s, n, h, w, 0))
        for p in P["blocks"]:
            cur, cur_s, h, w = self._block_cuda(p, cur, cur_s, n, h, w)
            if p["stage"] in self.out_indices:
                outs.append(self._stage(cur, cur_s, n, h, w, p["stage"]))
        if P["head"] is not None:
            cur = ops.gemm(cur_s, P["head"][0], bias=P["head"][1], act=3)
            outs.append(self._stage(cur, ops.to_split(cur), n, h, w, len(self.layers) - 1))
        return tuple(outs)

    @staticmethod
    def _block_cuda(p, x, x_s, n, h, w):
        """One InvertedResidual on the kernels: p = one entry of _prepare()["blocks"], x (n*h*w, Cinp) fp32 and its S32
        twin x_s (None when the block has no expand conv) -> (out fp32 (n*ho*wo, Coutp), its S32 twin or None, ho, wo)"""
        ks, st = p["k"], p["stride"]
        t = x if p["expand"] is None else ops.gemm(x_s, p["expand"][0], bias=p["expand"][1], act=3)
        ho, wo = -(-h // st), -(-w // st)
        y, part = ops.dwconv_swish(t.view(n, h, w, -1), *p["dw"], ks, st, adaptive_pad(h, ks, st)[0],
                                   adaptive_pad(w, ks, st)[0], ho, wo)
        gate = ops.se_gate(part, ho * wo, *p["se"])
        ys = ops.se_scale(y, gate).view(n * ho * wo, -1)
        out = ops.gemm(ys, p["linear"][0], bias=p["linear"][1], residual=x if p["res"] else None)
        return out, (ops.to_split(out) if p["split"] else None), ho, wo

    # ------------------------------------------------------------------ the torch restatement (CPU path, test oracle)
    def _forward_torch(self, x):
        outs = []
        for i, layer in enumerate(self.layers):
            x = layer(x)
            if i in self.out_indices:
                outs.append(x)
        return tuple(outs)
