"""Image encoder of the nuScenes R50 and R101 models: the stage in front of DepthNet that turns camera images into
feature maps.

    ResNet / Bottleneck      mmdet 2.14.0 mmdet/models/backbones/resnet.py (depth 50, style 'pytorch')
    ResNetDCN                the same ResNet at depth 50 / 101, style 'pytorch' / 'caffe', with DCNv2 3x3 convs
    ModulatedDeformConv2dPack  mmcv-full 1.4.0 mmcv/ops/modulated_deform_conv.py (the 'DCNv2' conv layer)
    SECONDFPN                mmdetection3d/mmdet3d/models/necks/second_fpn.py:11-91
    config                   projects/configs/occformer_nusc/occformer_nusc_r50_256x704.py:65-79 (img_backbone,
                             img_neck; the panoptic config uses the same two), occformer_nusc_r101_896x1600.py:67-84

Both modules take the reference's constructor kwargs and have its exact ``state_dict`` keys (ResNet's are torchvision's
``resnet50`` keys without ``fc.*``), so a reference checkpoint's ``img_backbone.*`` / ``img_neck.*`` entries load with
``strict=True``.  Inference only: BatchNorm uses its running statistics (eval mode).

On CUDA tensors ``forward`` runs on this package's sm_90a kernels (``_forward_cuda``, no host synchronisation, CUDA-graph
capturable).  Every convolution is the fp32-faithful GEMM / implicit-GEMM conv with the eval BatchNorms folded in once
per weight set (``_prepare``); the stem's im2col, the stem max-pool and SECONDFPN's pixel reshuffles are small kernels of
their own (csrc/image_ops.cu).  A CUDA input outside that path's shape contract raises RuntimeError; there is no cuDNN
fallback.  On CPU tensors ``forward`` is the plain torch restatement ``_forward_torch`` (the oracle of the GPU tests).

Stage outputs are handed on as the package's other module boundaries are: an fp32 NCHW view of channel-last memory
(torch's ``channels_last`` strides) carrying its S32 twin (common.attach_twin).  SECONDFPN picks the twin up while the
level is unmodified (common.twin_of), else it splits the level itself; its own output is
a ``channels_last`` map, which survives the reference glue's ``.view`` calls and which DepthNet splits without a
transpose.

``ResNet``, ``ResNetDCN`` and ``SECONDFPN`` are registered in this package's local registries only, never forced into
the upstream ones (INTEGRATION.md shows the opt-in).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .common import PreparedModule, attach_twin, batchnorm, fold_bn, round32, twin_of
from .depthnet import deform_columns
from .registry import BACKBONES, NECKS

# ---------------------------------------------------------------------------------------------------------- DCNv2
class ModulatedDeformConv2dPack(nn.Module):
    """mmcv-full 1.4.0 ``ModulatedDeformConv2dPack`` (mmcv/ops/modulated_deform_conv.py; the 'DCNv2' conv layer of mmdet's
    Bottleneck, built with bias=False): 3x3, stride 1, padding 1, dilation 1, groups 1, one deformable group.
    Parameters ``weight`` (out, in, 3, 3) and ``conv_offset`` = Conv2d(in, 27, 3, padding 1, bias).  Forward, as mmcv's:
    ``o1, o2, mask = chunk(conv_offset(x), 3, dim=1)``, ``offset = cat(o1, o2)``, ``mask = sigmoid(mask)``; kernel point
    k = ky*3 + kx takes (dy, dx) from offset channels 2k / 2k+1 and samples x at h = (y - 1 + ky) + dy, w = (x - 1 + kx) +
    dx, bilinear, zero unless h > -1 && w > -1 && h < H && w < W and each corner outside the map zero
    (modulated_deform_conv_cuda_kernel.cuh modulated_deformable_im2col_gpu_kernel / dmcn_im2col_bilinear); the column is
    val * mask_k, then the contraction with ``weight``.  Here the sampling is depthnet.deform_columns (``grid_sample``
    with zero padding, which zeroes every sample with h <= -1 or h >= H as mmcv's inside test does)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, dilation=1, groups=1,
                 deform_groups=1, bias=False):
        super().__init__()
        if kernel_size not in (3, (3, 3)) or (stride, padding, dilation, groups, deform_groups) != (1,) * 5 or bias:
            raise NotImplementedError("occformer_b200.ModulatedDeformConv2dPack: 3x3, stride 1, padding 1, dilation 1, "
                                      "groups 1, deform_groups 1, bias=False only")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, 3, 3))
        nn.init.kaiming_uniform_(self.weight, nonlinearity="relu")
        self.conv_offset = nn.Conv2d(in_channels, 27, 3, stride=1, padding=1, bias=True)
        nn.init.zeros_(self.conv_offset.weight)
        nn.init.zeros_(self.conv_offset.bias)

    def forward(self, x):
        C = x.shape[1]
        o1, o2, mask = torch.chunk(self.conv_offset(x), 3, dim=1)
        col = deform_columns(x, torch.cat((o1, o2), dim=1)) * torch.sigmoid(mask).unsqueeze(1)  # (B, C, 9, H, W)
        return torch.einsum("bckhw,ock->bohw", col, self.weight.view(self.out_channels, C, 9))


# ---------------------------------------------------------------------------------------------------------- ResNet
class Bottleneck(nn.Module):
    """mmdet Bottleneck: relu(bn3(conv3(relu(bn2(conv2(relu(bn1(conv1(x)))))))) + identity), identity = downsample(x) when
    present.  Style 'pytorch' puts the stride on the 3x3 conv2, style 'caffe' on the 1x1 conv1; dcn: conv2 is a
    ModulatedDeformConv2dPack (stride 1 only)."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, norm_cfg=None, style="pytorch", dcn=False):
        super().__init__()
        s1, s2 = (stride, 1) if style == "caffe" else (1, stride)
        self.conv1 = nn.Conv2d(inplanes, planes, 1, stride=s1, bias=False)
        self.bn1 = batchnorm(norm_cfg, planes, 1e-5)
        if dcn:
            assert s2 == 1
            self.conv2 = ModulatedDeformConv2dPack(planes, planes, 3, padding=1)
        else:
            self.conv2 = nn.Conv2d(planes, planes, 3, stride=s2, padding=1, bias=False)
        self.bn2 = batchnorm(norm_cfg, planes, 1e-5)
        self.conv3 = nn.Conv2d(planes, planes * self.expansion, 1, bias=False)
        self.bn3 = batchnorm(norm_cfg, planes * self.expansion, 1e-5)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride, self.style, self.dcn = stride, style, dcn

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(out))
        identity = x if self.downsample is None else self.downsample(x)
        return self.relu(out + identity)


@BACKBONES.register_module(upstream=False)
class ResNet(PreparedModule):
    """mmdet 2.14.0 ``ResNet`` at depth 50: forward(x (n, 3, H, W)) -> tuple of the stages in ``out_indices``, stage i
    with 64 * 2^(i+2) channels at stride 2^(i+2).

    Builds style 'pytorch', BatchNorm, strides (1, 2, 2, 2), dilation 1.  The training-only kwargs (frozen_stages,
    norm_eval, with_cp, zero_init_residual) and pretrained / init_cfg are accepted and ignored: construction does not
    touch the file system; load a checkpoint with load_state_dict.  Options this implementation does not have raise
    NotImplementedError naming the kwarg."""
    arch_settings = {50: (3, 4, 6, 3)}
    styles = ("pytorch",)
    scope = "depth 50, style 'pytorch', BatchNorm, strides (1, 2, 2, 2), dilation 1, plain stem"

    def __init__(self, depth, in_channels=3, stem_channels=None, base_channels=64, num_stages=4, strides=(1, 2, 2, 2),
                 dilations=(1, 1, 1, 1), out_indices=(0, 1, 2, 3), style="pytorch", deep_stem=False, avg_down=False,
                 frozen_stages=-1, conv_cfg=None, norm_cfg=dict(type="BN", requires_grad=True), norm_eval=True,
                 dcn=None, stage_with_dcn=(False, False, False, False), plugins=None, with_cp=False,
                 zero_init_residual=True, pretrained=None, init_cfg=None):
        super().__init__()

        def unsupported(kwarg, value):
            raise NotImplementedError(f"occformer_b200.{type(self).__name__}: {kwarg}={value!r} is not supported "
                                      f"({self.scope})")

        if depth not in self.arch_settings:
            unsupported("depth", depth)
        if style not in self.styles:
            unsupported("style", style)
        if deep_stem:
            unsupported("deep_stem", deep_stem)
        if avg_down:
            unsupported("avg_down", avg_down)
        self.stage_dcn = self._dcn_stages(dcn, stage_with_dcn, style, strides, num_stages, unsupported)
        if plugins:
            unsupported("plugins", plugins)
        if in_channels != 3:
            unsupported("in_channels", in_channels)
        if not 1 <= num_stages <= 4:
            unsupported("num_stages", num_stages)
        if tuple(strides[:num_stages]) != (1, 2, 2, 2)[:num_stages] or len(strides) != num_stages:
            unsupported("strides", strides)
        if tuple(dilations) != (1,) * num_stages:
            unsupported("dilations", dilations)
        if conv_cfg is not None and dict(conv_cfg).get("type", "Conv2d") not in ("Conv2d", "Conv"):
            unsupported("conv_cfg", conv_cfg)
        if any(not 0 <= i < num_stages for i in out_indices):
            unsupported("out_indices", out_indices)
        self.depth, self.num_stages, self.out_indices, self.style = depth, num_stages, tuple(out_indices), style
        self.base_channels = base_channels
        self.stem_channels = stem_channels or base_channels
        self.conv1 = nn.Conv2d(3, self.stem_channels, 7, stride=2, padding=3, bias=False)
        self.bn1 = batchnorm(norm_cfg, self.stem_channels, 1e-5)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.res_layers = []
        inplanes = self.stem_channels
        for i, blocks in enumerate(self.arch_settings[depth][:num_stages]):
            planes, stride = base_channels * 2 ** i, strides[i]
            downsample = None
            if stride != 1 or inplanes != planes * Bottleneck.expansion:
                downsample = nn.Sequential(nn.Conv2d(inplanes, planes * Bottleneck.expansion, 1, stride=stride, bias=False),
                                           batchnorm(norm_cfg, planes * Bottleneck.expansion, 1e-5))
            kw = dict(norm_cfg=norm_cfg, style=style, dcn=self.stage_dcn[i])
            layer = [Bottleneck(inplanes, planes, stride, downsample, **kw)]
            inplanes = planes * Bottleneck.expansion
            layer += [Bottleneck(inplanes, planes, 1, None, **kw) for _ in range(1, blocks)]
            self.add_module(f"layer{i + 1}", nn.Sequential(*layer))
            self.res_layers.append(f"layer{i + 1}")

    @staticmethod
    def _dcn_stages(dcn, stage_with_dcn, style, strides, num_stages, unsupported):
        """-> per stage whether its 3x3 convs are DCNv2; ResNet has none"""
        if dcn is not None:
            unsupported("dcn", dcn)
        if any(stage_with_dcn):
            unsupported("stage_with_dcn", stage_with_dcn)
        return (False,) * num_stages

    def forward(self, x):
        if x.is_cuda:
            return self._forward_cuda(x)
        return self._forward_torch(x)

    # ------------------------------------------------------------------ parameters of the CUDA forward
    @torch.no_grad()
    def _folded(self):
        """Eval BatchNorms folded into the convs before them (natural layouts, fp32 on the parameters' device):
        {"stem": (w (C0, 3, 7, 7), b), "blocks": [(stride, (w1, b1), (w2, b2), (w3, b3), (wd, bd) | None), ...]} with the
        blocks of all stages in order."""
        return {"stem": fold_bn(self.conv1.weight, None, self.bn1),
                "blocks": [self._fold_block(blk) for name in self.res_layers for blk in getattr(self, name)]}

    @staticmethod
    def _fold_block(blk):
        ds = blk.downsample
        return (blk.stride, fold_bn(blk.conv1.weight, None, blk.bn1), fold_bn(blk.conv2.weight, None, blk.bn2),
                fold_bn(blk.conv3.weight, None, blk.bn3), None if ds is None else fold_bn(ds[0].weight, None, ds[1]))

    @torch.no_grad()
    def _prepare(self):
        """The folded parameters in the kernels' layouts: the stem weight as a (C0, 160) S32 matrix in the im2col's
        (ky, kx, c) column order (zero columns 147..159), the block convs repacked tap-major in S32."""
        F_ = self._folded()
        w, b = F_["stem"]
        wm = w.permute(0, 2, 3, 1).reshape(w.shape[0], 147)
        wm = torch.cat([wm, wm.new_zeros(w.shape[0], ops.STEM_COLS - 147)], dim=1)
        return {"stem": (ops.split_weight(wm), b), "blocks": [self._prepare_block(fb) for fb in F_["blocks"]]}

    @staticmethod
    def _repack(wb):
        return None if wb is None else (ops.repack_conv_weight(wb[0])[0], wb[1])

    @classmethod
    def _prepare_block(cls, fb):
        s, c1, c2, c3, d = fb
        return (s, cls._repack(c1), cls._repack(c2), cls._repack(c3), cls._repack(d))

    def _check_cuda_contract(self, x):
        need = []
        if x.dim() != 4 or x.shape[1] != 3:
            need.append("x of shape (n, 3, H, W)")
        elif x.shape[2] % 32 or x.shape[3] % 32:
            need.append("H and W multiples of 32 (every stage size exact)")
        if self.stem_channels % 32 or self.base_channels % 32:
            need.append("stem_channels and base_channels multiples of 32 (whole 32-channel chunks of the conv operands)")
        if x.dim() == 4 and x.shape[0] > 65535:
            need.append("n <= 65535")
        if self.training:
            need.append("eval mode (the CUDA forward applies the BatchNorms' running statistics; call .eval())")
        if need:
            raise RuntimeError(f"occformer_b200: {type(self).__name__}'s CUDA forward needs {'; '.join(need)} -- got x "
                               f"{tuple(x.shape)}, "
                               f"stem_channels {self.stem_channels}, base_channels {self.base_channels}")

    @torch.no_grad()
    def _forward_cuda(self, x):
        self._check_cuda_contract(x)
        P = self.prepared()
        n, _, H, W = x.shape
        stem = ops.gemm(ops.stem_im2col(x.float().contiguous()), P["stem"][0], bias=P["stem"][1], act=1)
        cur_s = ops.maxpool3x3s2(stem.view(n, H // 2, W // 2, -1)).unsqueeze(3)  # (n, H/4, W/4, 1, C0) S32
        cur = None  # fp32 twin of the block input (the stem's is never needed: layer1.0 has a downsample)
        outs, i = [], 0
        for si, name in enumerate(self.res_layers):
            for _ in getattr(self, name):
                cur, cur_s = self._bottleneck_cuda(P["blocks"][i], cur, cur_s)
                i += 1
            if si in self.out_indices:
                nn_, h, w, _, C = cur.shape
                v = cur.view(nn_, h, w, C).permute(0, 3, 1, 2)  # NCHW view, channels_last strides
                outs.append(attach_twin(v, cur_s.view(nn_, h, w, C)))
        return tuple(outs)

    @staticmethod
    def _bottleneck_cuda(p, x, x_s):
        """One Bottleneck on the kernels: p = one entry of _prepare()["blocks"], x (n, h, w, 1, C) fp32 (may be None when
        the block has a downsample) and its S32 twin x_s -> (out fp32, out S32), each (n, h/s, w/s, 1, 4 * planes)."""
        s, (w1, b1), (w2, b2), (w3, b3), ds = p
        k1, k3 = (1, 1, 1), (3, 3, 1)
        t = ops.conv(x_s, w1, k1, bias=b1, act=1, split_out=True)
        t = ops.conv(t, w2, k3, stride=s, bias=b2, act=1, split_out=True)
        ident = x if ds is None else ops.conv(x_s, ds[0], k1, stride=s, bias=ds[1])
        out = ops.conv(t, w3, k1, bias=b3, residual=ident, act=1)  # relu(bn3(conv3) + identity)
        return out, ops.to_split(out)

    # ------------------------------------------------------------------ the torch restatement (CPU path, test oracle)
    def _forward_torch(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        outs = []
        for i, name in enumerate(self.res_layers):
            x = getattr(self, name)(x)
            if i in self.out_indices:
                outs.append(x)
        return tuple(outs)


@BACKBONES.register_module(upstream=False)
class ResNetDCN(ResNet):
    """mmdet 2.14.0 ``ResNet`` with the options of the nuScenes R101 config (occformer_nusc_r101_896x1600.py:68-79): depth
    50 or 101, style 'pytorch' or 'caffe' (mmdet's Bottleneck puts the stage stride on conv1 in caffe style), and
    ``dcn=dict(type='DCNv2', deform_groups=1, fallback_on_stride=False)`` on the stages of ``stage_with_dcn``, whose 3x3
    conv2 is then a ModulatedDeformConv2dPack.  A DCN on a strided conv2 (style 'pytorch', stages 2-4) is not supported;
    everything else is ResNet's: same keys (plus ``layer{i}.{j}.conv2.conv_offset.{weight,bias}``), same kwargs, the
    same NotImplementedError for the options neither has.  ``norm_cfg`` type 'BN2d' is BatchNorm.

    CUDA forward of a DCN Bottleneck: conv1 (1x1, stride s in caffe style, S32 out) -> conv_offset (3x3 conv, Cout
    padded 27 -> 32, fp32 rows) -> ops.modulated_deform_im2col -> GEMM of the columns with the tap-major conv2 weight (bn2
    folded, ReLU, S32 out) -> conv3 + identity + ReLU -> split: two launches more than a plain Bottleneck."""
    arch_settings = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}
    styles = ("pytorch", "caffe")
    scope = ("depth 50 or 101, style 'pytorch' or 'caffe', dcn DCNv2 with deform_groups 1 and fallback_on_stride "
             "False on stride-1 3x3 convs only (a DCN in stages 2-4 needs style 'caffe'), BatchNorm, strides (1, 2, 2, 2), "
             "dilation 1, plain stem")

    @staticmethod
    def _dcn_stages(dcn, stage_with_dcn, style, strides, num_stages, unsupported):
        if dcn is None:  # mmdet: stage_with_dcn only matters with a dcn
            return (False,) * num_stages
        d = dict(dcn)
        if d.get("type") != "DCNv2" or d.get("deform_groups", 1) != 1 or d.get("fallback_on_stride", False) or \
                set(d) - {"type", "deform_groups", "fallback_on_stride"}:
            unsupported("dcn", dcn)
        if len(stage_with_dcn) != num_stages:
            unsupported("stage_with_dcn", stage_with_dcn)
        if style != "caffe" and any(w and s != 1 for w, s in zip(stage_with_dcn, strides)):
            unsupported("stage_with_dcn", stage_with_dcn)
        return tuple(bool(w) for w in stage_with_dcn)

    @staticmethod
    def _fold_block(blk):
        """ResNet's block entry + (caffe, conv_offset (w (32, C, 3, 3), b (32)) zero-padded from 27 channels | None)"""
        off = None
        if blk.dcn:
            co = blk.conv2.conv_offset
            w, b = co.weight.detach().float(), co.bias.detach().float()
            off = (torch.cat([w, w.new_zeros(32 - w.shape[0], *w.shape[1:])]).contiguous(),
                   torch.cat([b, b.new_zeros(32 - b.shape[0])]).contiguous())
        return ResNet._fold_block(blk) + (blk.style == "caffe", off)

    @classmethod
    def _prepare_block(cls, fb):
        return super()._prepare_block(fb[:5]) + (fb[5], cls._repack(fb[6]))

    @staticmethod
    def _bottleneck_cuda(p, x, x_s):
        """ResNet._bottleneck_cuda for an entry of ResNetDCN._prepare()["blocks"]: stride on conv1 when caffe, conv2 a
        DCNv2 when the entry has conv_offset weights."""
        s, (w1, b1), (w2, b2), (w3, b3), ds, caffe, off = p
        s1, s2 = (s, 1) if caffe else (1, s)
        k1, k3 = (1, 1, 1), (3, 3, 1)
        t = ops.conv(x_s, w1, k1, stride=s1, bias=b1, act=1, split_out=True)
        if off is None:
            t = ops.conv(t, w2, k3, stride=s2, bias=b2, act=1, split_out=True)
        else:
            n, h, w, _, C = t.shape
            o = ops.conv(t, off[0], k3, bias=off[1]).view(n * h * w, 32)
            cols = ops.modulated_deform_im2col(t, o, n, h, w)
            t = ops.gemm(cols, w2, bias=b2, act=1, split_out=True).view(n, h, w, 1, C)
        ident = x if ds is None else ops.conv(x_s, ds[0], k1, stride=s, bias=ds[1])
        out = ops.conv(t, w3, k1, bias=b3, residual=ident, act=1)
        return out, ops.to_split(out)


# ---------------------------------------------------------------------------------------------------------- SECONDFPN
@NECKS.register_module(upstream=False)
class SECONDFPN(PreparedModule):
    """second_fpn.py:11-91: one deblock per level -- ConvTranspose2d(kernel = stride = s) for an upsample stride s >= 1
    (s == 1 also Conv2d(1x1) with use_conv_for_no_stride), Conv2d(kernel = stride = 1/s) for s < 1 -- each followed by
    BatchNorm (default eps 1e-3) and ReLU; forward(levels) -> [channel concat of the deblock outputs].  On CUDA a level
    whose width is not a multiple of 32 must carry its zero-padded S32 twin and be unmodified since
    (CustomEfficientNet's stages are handed over so)."""

    def __init__(self, in_channels=[128, 128, 256], out_channels=[256, 256, 256], upsample_strides=[1, 2, 4],
                 norm_cfg=dict(type="BN", eps=1e-3, momentum=0.01), upsample_cfg=dict(type="deconv", bias=False),
                 conv_cfg=dict(type="Conv2d", bias=False), use_conv_for_no_stride=False, init_cfg=None):
        super().__init__()
        assert len(out_channels) == len(upsample_strides) == len(in_channels)
        up, cv = dict(upsample_cfg), dict(conv_cfg)
        if up.pop("type", "deconv") != "deconv":
            raise NotImplementedError(f"occformer_b200.SECONDFPN: upsample_cfg={upsample_cfg!r} is not supported "
                                      "(deconv only)")
        if cv.pop("type", "Conv2d") not in ("Conv2d", "Conv"):
            raise NotImplementedError(f"occformer_b200.SECONDFPN: conv_cfg={conv_cfg!r} is not supported (Conv2d only)")
        self.in_channels, self.out_channels = list(in_channels), list(out_channels)
        self.upsample_strides = list(upsample_strides)
        deblocks = []
        for i, out_channel in enumerate(out_channels):
            stride = upsample_strides[i]
            if stride > 1 or (stride == 1 and not use_conv_for_no_stride):
                k = int(stride)
                layer = nn.ConvTranspose2d(in_channels[i], out_channel, kernel_size=k, stride=k, **up)
            else:
                k = int(round(1 / stride))
                layer = nn.Conv2d(in_channels[i], out_channel, kernel_size=k, stride=k, **cv)
            deblocks.append(nn.Sequential(layer, batchnorm(norm_cfg, out_channel, 1e-5), nn.ReLU(inplace=True)))
        self.deblocks = nn.ModuleList(deblocks)

    def forward(self, x):
        assert len(x) == len(self.in_channels)
        if x[0].is_cuda:
            return self._forward_cuda(x)
        return self._forward_torch(x)

    # ------------------------------------------------------------------ parameters of the CUDA forward
    @torch.no_grad()
    def _folded(self):
        """Per deblock (kind, f, w, b) with the BatchNorm folded in (natural layouts, fp32): kind "conv" = Conv2d
        kernel = stride = f, w (Cout, Cin, f, f); kind "deconv" = ConvTranspose2d kernel = stride = f, w (Cin, Cout, f,
        f)."""
        res = []
        for blk in self.deblocks:
            layer, bn = blk[0], blk[1]
            deconv = isinstance(layer, nn.ConvTranspose2d)
            w, b = fold_bn(layer.weight, layer.bias, bn, out_dim=1 if deconv else 0)
            res.append(("deconv" if deconv else "conv", layer.stride[0], w, b))
        return res

    @torch.no_grad()
    def _prepare(self):
        """The kernels' layouts: a conv (or a 1x1 deconv) as a tap-major S32 (Cout, f*f*Cin) matrix, the operand of a 1x1
        conv of the space_to_depth'd input; a stride-f deconv as the S32 (f*f*Cout, Cin) matrix whose row (i*f + j)*Cout
        + o is w[:, o, i, j], with its bias repeated per (i, j)."""
        P = []
        for (kind, f, w, b), cin in zip(self._folded(), self.in_channels):
            pad = round32(cin) - cin  # zero input columns (per tap) for a level whose S32 twin is zero-padded
            if kind == "conv":
                P.append(("down", f, ops.repack_conv_weight(F.pad(w, (0, 0, 0, 0, 0, pad)))[0], b))
            elif f == 1:
                P.append(("down", 1, ops.split_weight(F.pad(w[:, :, 0, 0].t(), (0, pad))), b))
            else:
                P.append(("up", f, ops.split_weight(F.pad(w.permute(2, 3, 1, 0).reshape(-1, w.shape[0]), (0, pad))),
                          b.repeat(f * f)))
        return P

    def _out_size(self, x):
        sizes = set()
        for t, s in zip(x, self.upsample_strides):
            H, W = t.shape[-2:]
            sizes.add((H * s, W * s))
        return sizes

    def _check_cuda_contract(self, x):
        need = []
        if any(t.dim() != 4 or t.shape[1] != c for t, c in zip(x, self.in_channels)):
            need.append(f"levels of shape (n, C_i, H_i, W_i) with C_i = {self.in_channels}")
        if any(c % 32 for c in self.out_channels) or (not need and any(
                c % 32 and twin_of(t) is None for t, c in zip(x, self.in_channels))):
            need.append("in_channels and out_channels multiples of 32 (whole 32-channel chunks; a narrower level must "
                        "carry its S32 twin zero-padded to whole chunks, as CustomEfficientNet hands it over, and be "
                        "unmodified since)")
        if any(s not in (0.25, 0.5, 1, 2, 4) for s in self.upsample_strides):
            need.append("upsample_strides in {0.25, 0.5, 1, 2, 4}")
        if not need:
            hw = [t.shape[-2:] for t in x]
            if any(h * s != int(h * s) or w * s != int(w * s) for (h, w), s in zip(hw, self.upsample_strides)) or \
                    len(self._out_size(x)) != 1 or len({t.shape[0] for t in x}) != 1:
                need.append("level sizes that the upsample strides map to one output size (H_i * s_i equal for all i, "
                            "exact) and one batch")
            elif x[0].shape[0] > 65535:
                need.append("n <= 65535")
        if self.training:
            need.append("eval mode (the CUDA forward applies the BatchNorms' running statistics; call .eval())")
        if need:
            raise RuntimeError(f"occformer_b200: SECONDFPN's CUDA forward needs {'; '.join(need)} -- got levels "
                               f"{[tuple(t.shape) for t in x]}, upsample_strides {self.upsample_strides}")

    @torch.no_grad()
    def _forward_cuda(self, x):
        self._check_cuda_contract(x)
        P = self.prepared()
        n = x[0].shape[0]
        Ho, Wo = (int(v) for v in next(iter(self._out_size(x))))
        out = torch.empty((n * Ho * Wo, sum(self.out_channels)), dtype=torch.float32, device=x[0].device)
        off = 0
        for t, (kind, f, w, b), cout in zip(x, P, self.out_channels):
            _, C, H, W = t.shape
            t_s = twin_of(t)
            if t_s is None:
                t_s = ops.split_nchw(t.float())
            C = t_s.shape[-1]
            if kind == "down":
                if f > 1:
                    t_s = ops.space_to_depth(t_s, f)
                ops.conv_into(t_s.view(n, Ho, Wo, 1, -1), w, (1, 1, 1), out, off, bias=b, act=1)
            else:
                y = ops.gemm(t_s.view(n * H * W, C), w, bias=b, act=1)
                ops.depth_to_space_into(y, n, H, W, f, out, off)
            off += cout
        return [out.view(n, Ho, Wo, off).permute(0, 3, 1, 2)]

    # ------------------------------------------------------------------ the torch restatement (CPU path, test oracle)
    def _forward_torch(self, x):
        ups = [deblock(x[i]) for i, deblock in enumerate(self.deblocks)]
        return [torch.cat(ups, dim=1) if len(ups) > 1 else ups[0]]
