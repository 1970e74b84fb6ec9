"""H100-native dual-path voxel transformer encoder, drop-in for the reference's modules:

    BACKBONES 'OccupancyEncoder'              projects/mmdet3d_plugin/occformer/backbones/occnet.py:12-74
    DualpathTransformerBlock                  .../backbones/dualpath_block.py:13-82
    SwinBlock / ShiftWindowMSA / WindowMSA    .../backbones/modules/window_attention.py:14-372
    BottleNeckASPP / ASPP                     .../backbones/modules/aspp.py:49-172

Same constructor kwargs, same ``forward(x (B,C,X,Y,Z)) -> list[Tensor (B,C,X',Y',Z')]``, same ``state_dict``
keys and shapes (SURVEY.md Appendix B) -- the torch.nn sub-modules below are *parameter containers only*;
all arithmetic runs in libocc_b200.so (wgmma GEMM / implicit-GEMM conv on split-bf16 operands -- three tensor-core
passes per contraction, fp32-faithful --, fused norm / window attention / fusion kernels).  Inference (eval, no
autograd) only.  Internally every tensor is channel-last (B,X,Y,Z,C); tensors that feed a tensor-core contraction are
kept in the S32 split format (ops.py); returned tensors are fp32 permuted *views* with the reference's shape that carry
their S32 twin (common.attach_twin; the next module of this package picks it up instead of re-splitting).
"""
import torch
import torch.nn as nn

from . import ops
from .common import PreparedModule, attach_twin, twin_of
from .registry import BACKBONES


def _gn(norm_cfg, channels, groups=None):
    g = groups if groups is not None else norm_cfg.get("num_groups", 32)
    return nn.GroupNorm(g, channels, eps=1e-5)


class _WindowMSA(nn.Module):
    def __init__(self, embed_dims, num_heads, ws=7):
        super().__init__()
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws - 1) * (2 * ws - 1), num_heads))
        seq1 = torch.arange(0, (2 * ws - 1) * ws, 2 * ws - 1)
        seq2 = torch.arange(0, ws, 1)
        c = (seq1[:, None] + seq2[None, :]).reshape(1, -1)
        self.register_buffer("relative_position_index", (c + c.T).flip(1).contiguous())
        self.qkv = nn.Linear(embed_dims, embed_dims * 3, bias=True)
        self.proj = nn.Linear(embed_dims, embed_dims)
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)


class _ShiftWindowMSA(nn.Module):
    def __init__(self, embed_dims, num_heads):
        super().__init__()
        self.w_msa = _WindowMSA(embed_dims, num_heads)


class _FFN(nn.Module):
    def __init__(self, embed_dims, hidden):
        super().__init__()
        self.layers = nn.Sequential(nn.Sequential(nn.Linear(embed_dims, hidden), nn.GELU(), nn.Dropout(0.0)),
                                    nn.Linear(hidden, embed_dims), nn.Dropout(0.0))


class _SwinBlock(nn.Module):
    def __init__(self, embed_dims, num_heads, shift):
        super().__init__()
        self.shift = shift
        self.num_heads = num_heads
        self.norm1 = nn.LayerNorm(embed_dims)
        self.attn = _ShiftWindowMSA(embed_dims, num_heads)
        self.norm2 = nn.LayerNorm(embed_dims)
        self.ffn = _FFN(embed_dims, embed_dims)


class _ASPPModule(nn.Module):
    def __init__(self, inplanes, planes, k, dilation, groups):
        super().__init__()
        self.atrous_conv = nn.Conv2d(inplanes, planes, k, stride=1, padding=0 if k == 1 else dilation,
                                     dilation=dilation, bias=False)
        self.bn = nn.GroupNorm(groups, planes)
        nn.init.kaiming_normal_(self.atrous_conv.weight)


class _ASPP(nn.Module):
    def __init__(self, ch, dilations, groups):
        super().__init__()
        self.aspp1 = _ASPPModule(ch, ch, 1, dilations[0], groups)
        self.aspp2 = _ASPPModule(ch, ch, 3, dilations[1], groups)
        self.aspp3 = _ASPPModule(ch, ch, 3, dilations[2], groups)
        self.aspp4 = _ASPPModule(ch, ch, 3, dilations[3], groups)
        self.global_avg_pool = nn.Sequential(nn.AdaptiveAvgPool2d((1, 1)), nn.Conv2d(ch, ch, 1, bias=False),
                                             nn.GroupNorm(groups, ch), nn.ReLU())
        self.conv1 = nn.Conv2d(5 * ch, ch, 1, bias=False)
        self.bn1 = nn.GroupNorm(groups, ch)
        nn.init.kaiming_normal_(self.conv1.weight)
        nn.init.kaiming_normal_(self.global_avg_pool[1].weight)


class _BottleNeckASPP(nn.Module):
    def __init__(self, inplanes, norm_cfg, reduction=4, dilations=(1, 6, 12, 18)):
        super().__init__()
        ch = inplanes // reduction
        ng = norm_cfg.get("num_groups", 32)
        self.dilations = tuple(dilations)
        self.inner_groups = ch // 2 if ch <= ng else ng  # aspp.py:150-154
        self.outer_groups = ng
        self.input_conv = nn.Sequential(nn.Conv2d(inplanes, ch, 1, bias=False), nn.GroupNorm(ng, ch), nn.ReLU())
        self.aspp = _ASPP(ch, dilations, self.inner_groups)
        self.output_conv = nn.Sequential(nn.Conv2d(ch, inplanes, 1, bias=False), nn.GroupNorm(ng, inplanes), nn.ReLU())


class DualpathTransformerBlock(PreparedModule):
    """dualpath_block.py:13-82.  ``layer_index`` decides the window shift (odd = shifted)."""

    def __init__(self, in_channels, channels, stride=1, norm_cfg=None, init_cfg=None, coeff_bias=True, aspp_drop=0.1,
                 **kwargs):
        super().__init__()
        norm_cfg = dict(norm_cfg or dict(type="GN", num_groups=32))
        assert norm_cfg.get("type", "GN") == "GN", "the CUDA path implements the reference's GN configuration"
        self.in_channels, self.channels, self.stride = in_channels, channels, stride
        self.groups = norm_cfg.get("num_groups", 32)
        self.shift = (kwargs["layer_index"] % 2) == 1
        self.num_heads = int(channels / 32)
        if stride > 1:
            self.downsample = nn.Sequential(nn.Conv3d(in_channels, channels, 1, stride=stride, bias=False),
                                            _gn(norm_cfg, channels))
        else:
            self.downsample = nn.Identity()
        self.input_conv = nn.Sequential(nn.Conv3d(in_channels, channels, 3, padding=1, stride=stride, bias=False),
                                        _gn(norm_cfg, channels), nn.ReLU())
        self.bev_encoder = _SwinBlock(channels, self.num_heads, self.shift)
        self.aspp = _BottleNeckASPP(channels, norm_cfg)
        self.combine_coeff = nn.Conv3d(channels, 1, 1, bias=coeff_bias)

    # ------------------------------------------------------------------ one-time weight preparation
    @torch.no_grad()
    def _prepare(self):
        sw_ = ops.split_weight
        P = {}
        P["w_in"], P["k_in"] = ops.repack_conv_weight(self.input_conv[0].weight)
        if self.stride > 1:
            P["w_ds"], P["k_ds"] = ops.repack_conv_weight(self.downsample[0].weight)
        msa = self.bev_encoder.attn.w_msa
        # qkv rows permuted to [head][q|k|v][32]: one S32 chunk per (token, head, q|k|v), the three chunks of a head
        # adjacent -- the attention kernel reads one contiguous 384-byte run per (token, head)
        perm = ops.qkv_head_major_perm(msa.qkv.weight.shape[1], self.num_heads, msa.qkv.weight.device)
        P["w_qkv"] = sw_(msa.qkv.weight.detach().float()[perm])
        P["b_qkv"] = msa.qkv.bias.detach().float()[perm].clone().contiguous()
        P["b_qkv_s"] = sw_(P["b_qkv"].view(1, -1)).view(-1)  # q/k/v of the zero pad tokens, as the kernel's operand rows
        P["w_proj"] = sw_(msa.proj.weight)
        ffn = self.bev_encoder.ffn.layers
        P["w_f1"] = sw_(ffn[0][0].weight)
        P["w_f2"] = sw_(ffn[1].weight)
        table = msa.relative_position_bias_table.detach().float()
        idx = msa.relative_position_index.view(-1)
        dense = table[idx].view(49, 49, -1).permute(2, 0, 1).reshape(-1, 49 * 49)  # (heads, 49*49)
        P["bias_pad"] = torch.nn.functional.pad(dense, (0, 2404 - 49 * 49)).contiguous()  # 16-byte multiple per head
        a = self.aspp
        P["w_a_in"], P["k1"] = ops.repack_conv_weight(a.input_conv[0].weight)
        for i in (1, 2, 3, 4):
            P[f"w_a{i}"], P[f"k_a{i}"] = ops.repack_conv_weight(getattr(a.aspp, f"aspp{i}").atrous_conv.weight)
        # the four ASPP branches (1x1 + three dilated 3x3 on the same input) as ONE tap-table convolution when their
        # 4 * inner_groups GroupNorm groups fit the conv epilogue's statistics (stage 0: 4 x 16): taps = centre + 8 x 3 rings
        ch = a.input_conv[0].weight.shape[0]
        P["aspp_merged"] = None
        ks = [tuple(getattr(a.aspp, f"aspp{i}").atrous_conv.weight.shape[-2:]) for i in (1, 2, 3, 4)]
        if 4 * a.inner_groups <= 64 and ks == [(1, 1), (3, 3), (3, 3), (3, 3)] and ch % 32 == 0:
            taps = [(0, 0, 0)]
            for d in a.dilations[1:]:
                taps += [(i * d, j * d, 0) for i in (-1, 0, 1) for j in (-1, 0, 1) if (i, j) != (0, 0)]
            wm = torch.zeros(4 * ch, len(taps), ch)
            wm[0:ch, 0] = a.aspp.aspp1.atrous_conv.weight.detach().float().cpu()[:, :, 0, 0]
            for bi, d in enumerate(a.dilations[1:], start=1):
                wb = getattr(a.aspp, f"aspp{bi + 1}").atrous_conv.weight.detach().float().cpu()  # (ch, ch, 3, 3) [kx][ky]
                for i in (-1, 0, 1):
                    for j in (-1, 0, 1):
                        t = 0 if (i, j) == (0, 0) else taps.index((i * d, j * d, 0))
                        wm[bi * ch:(bi + 1) * ch, t] = wb[:, :, i + 1, j + 1]
            dev = a.input_conv[0].weight.device
            gns = [getattr(a.aspp, f"aspp{i}").bn for i in (1, 2, 3, 4)]
            P["aspp_merged"] = dict(taps=taps, w=ops.split_weight(wm.reshape(4 * ch, -1)).to(dev),
                                    gw=torch.cat([g.weight.detach().float() for g in gns]).contiguous(),
                                    gb=torch.cat([g.bias.detach().float() for g in gns]).contiguous())
        P["w_gap"] = a.aspp.global_avg_pool[1].weight.detach().float().reshape(a.aspp.global_avg_pool[1].weight.shape[0], -1).contiguous()
        P["w_a_c1"], _ = ops.repack_conv_weight(a.aspp.conv1.weight)
        P["w_a_out"], _ = ops.repack_conv_weight(a.output_conv[0].weight)
        P["coeff_w"] = self.combine_coeff.weight.detach().float().reshape(-1).contiguous()
        P["coeff_b"] = float(self.combine_coeff.bias.detach().float().item()) if self.combine_coeff.bias is not None else 0.0
        return P

    # ------------------------------------------------------------------ forward on channel-last tensors
    @torch.no_grad()
    def forward_cl(self, x_cl, x_s=None, want_f32=True):
        """x_cl (B,X,Y,Z,Cin) contiguous channel-last fp32 (may be None when its S32 twin x_s is given)
        -> (out fp32 (B,X',Y',Z',C) | None, out S32): the S32 output feeds the next block / the neck, the fp32 one is
        only produced when the caller wants it (stage outputs)."""
        P = self.prepared()
        if x_s is None:
            x_s = ops.to_split(x_cl)
        B, X0, Y0, Z0, Cin = x_s.shape
        C, G, s = self.channels, self.groups, self.stride
        dev = x_s.device
        stats = torch.zeros((10, B, 64, 2), dtype=torch.float64, device=dev)
        # (A4) Conv3d 3x3x3 (+stride) -> raw output + GroupNorm statistics from the GEMM epilogue
        y_raw = ops.conv(x_s, P["w_in"], P["k_in"], stride=s, gn_stats=stats[0], cpg=C // G)
        _, X, Y, Z, _ = y_raw.shape
        XY = X * Y
        nvox = B * XY * Z
        ic, sw = self.input_conv, self.bev_encoder
        # (A4/A5/A6) GN + ReLU, Z-mean BEV token, LayerNorm1 -- one pass; tok fp32 (residual), tokn S32 (GEMM operand)
        # (at C == 128 tokn is written straight into the window layout the fused attention kernel loads by TMA)
        tok, tokn = ops.gn_relu_zmean_ln(y_raw.view(nvox, C), stats[0], ic[1].weight, ic[1].bias, sw.norm1.weight,
                                         sw.norm1.bias, B, XY, Z, C, G, X=X, win_shift=self.shift if C == 128 else None)
        msa = sw.attn.w_msa
        if C == 128:
            # (A7/A8) QKV projection + shifted-window attention in one kernel: the qkv tensor never exists in HBM
            att = ops.swin_qkv_attention(tokn, P["w_qkv"], P["b_qkv"], P["bias_pad"], B, X, Y, Z, C, self.num_heads, self.shift)
        else:
            # (A8) QKV projection of every token (pad tokens are synthesised from the bias inside the attention kernel)
            qkv = ops.gemm(tokn, P["w_qkv"], bias=P["b_qkv"], split_out=True)
            # (A7/A8) shifted-window attention core, gathers/scatters windows in place
            att = ops.window_attention(qkv, P["b_qkv_s"], P["bias_pad"], B, X, Y, Z, C, self.num_heads, self.shift,
                                       head_major=True)
        # proj + residual, LayerNorm2, FFN (GELU) + residual  (A6)
        ffn = sw.ffn.layers
        if C == 128 and P["w_f1"].shape == (C, C):
            # one kernel: the three 128x128 GEMMs are chained through registers, y1 / LN2(y1) / h never reach HBM
            y2 = ops.swin_proj_ffn(att, tok, P["w_proj"], msa.proj.bias, sw.norm2.weight, sw.norm2.bias, P["w_f1"],
                                   ffn[0][0].bias, P["w_f2"], ffn[1].bias)
        else:
            y1 = ops.gemm(att, P["w_proj"], bias=msa.proj.bias, residual=tok)
            y1n = ops.layernorm(y1, sw.norm2.weight, sw.norm2.bias, split_out=True)
            h = ops.gemm(y1n, P["w_f1"], bias=ffn[0][0].bias, act=2, split_out=True)
            y2 = ops.gemm(h, P["w_f2"], bias=ffn[1].bias, residual=y1)
        x_vox, x_bev = y2[:nvox], y2[nvox:]
        # (A9) BottleNeckASPP on the BEV tokens (B, X, Y, 1, C)
        bev_out = self._aspp(x_bev, B, X, Y, C, stats, P)
        # (A10) fusion + skip connection
        if s > 1:
            id_raw = ops.conv(x_s, P["w_ds"], P["k_ds"], stride=s, gn_stats=stats[9], cpg=C // G)
            out, out_s = ops.dualpath_fuse(x_vox, bev_out, P["coeff_w"], P["coeff_b"], id_raw.view(nvox, C), B, XY, Z, C,
                                           id_stats=stats[9], id_w=self.downsample[1].weight,
                                           id_b=self.downsample[1].bias, groups=G, want_f32=want_f32)
        else:
            out, out_s = ops.dualpath_fuse(x_vox, bev_out, P["coeff_w"], P["coeff_b"], x_s.view(nvox, C), B, XY, Z, C,
                                           identity_split=True, want_f32=want_f32)
        return (out.view(B, X, Y, Z, C) if out is not None else None), out_s.view(B, X, Y, Z, C)

    def _aspp(self, x_bev, B, X, Y, C, stats, P):
        a = self.aspp
        ch = C // 4
        XY = X * Y
        gi, go = a.inner_groups, a.outer_groups

        def conv2d(t_s, w, k, dil=1, st=None, cpg=0):
            cin = t_s.shape[-1]
            return ops.conv(t_s.view(B, X, Y, 1, cin), w, k, dil=dil, gn_stats=st, cpg=cpg).view(B * XY, -1)

        t = conv2d(ops.to_split(x_bev), P["w_a_in"], (1, 1, 1), st=stats[1], cpg=ch // go)
        y, y_s = ops.gn_apply(t, stats[1], a.input_conv[1].weight, a.input_conv[1].bias, XY, go, want_split=True)
        cat_s = torch.empty((B * XY, 5 * ch), dtype=torch.float32, device=x_bev.device)  # S32 concat buffer
        mg = P["aspp_merged"]
        if mg is not None:
            # all four branches in one 25-tap launch; their GroupNorms are one GroupNorm(4 * gi groups) over 4 * ch channels
            t = ops.conv_taps(y_s.view(B, X, Y, 1, ch), mg["w"], mg["taps"], gn_stats=stats[2].view(-1)[:B * 4 * gi * 2].view(B, 4 * gi, 2),
                              cpg=ch // gi).view(B * XY, 4 * ch)
            ops.gn_apply(t, stats[2].view(-1)[:B * 4 * gi * 2].view(B, 4 * gi, 2), mg["gw"], mg["gb"], XY, 4 * gi, want_f32=False,
                         split_into=cat_s, out_off=0)
        for i, d in zip((1, 2, 3, 4) if mg is None else (), a.dilations):
            m = getattr(a.aspp, f"aspp{i}")
            k = P[f"k_a{i}"]
            t = conv2d(y_s, P[f"w_a{i}"], k, dil=d if k[0] == 3 else 1, st=stats[1 + i], cpg=ch // gi)
            ops.gn_apply(t, stats[1 + i], m.bn.weight, m.bn.bias, XY, gi, want_f32=False, split_into=cat_s,
                         out_off=(i - 1) * ch)
        gap = a.aspp.global_avg_pool
        ops.aspp_gap_branch(y, P["w_gap"], gap[2].weight, gap[2].bias, cat_s, B, XY, gi, 4 * ch)
        t = conv2d(cat_s, P["w_a_c1"], (1, 1, 1), st=stats[6], cpg=ch // gi)
        _, y3_s = ops.gn_apply(t, stats[6], a.aspp.bn1.weight, a.aspp.bn1.bias, XY, gi, residual=y, want_f32=False,
                               want_split=True)
        t = conv2d(y3_s, P["w_a_out"], (1, 1, 1), st=stats[7], cpg=C // go)
        bev_out, _ = ops.gn_apply(t, stats[7], a.output_conv[1].weight, a.output_conv[1].bias, XY, go, residual=x_bev)
        return bev_out

    def forward(self, x):
        out, out_s = self.forward_cl(*to_channel_last(x))
        return to_reference_layout(out, out_s)


def to_channel_last(x):
    """(B,C,X,Y,Z) reference-layout tensor (any strides) -> (contiguous (B,X,Y,Z,C) fp32, its S32 twin or None).
    Zero-copy when x is already a permuted view of channel-last memory (what this package's own modules hand around);
    the S32 twin is the one such a view carries (common.twin_of)."""
    if not x.is_cuda:
        raise RuntimeError("occformer_b200: the encoder runs on CUDA tensors only (no CPU fallback)")
    return x.float().permute(0, 2, 3, 4, 1).contiguous(), twin_of(x)


def to_reference_layout(x_cl, x_s=None):
    """channel-last (B,X,Y,Z,C) -> the reference's (B,C,X,Y,Z) as a permuted view; the S32 twin rides along."""
    v = x_cl.permute(0, 4, 1, 2, 3)
    return v if x_s is None else attach_twin(v, x_s)


@BACKBONES.register_module()
class OccupancyEncoder(nn.Module):
    """occnet.py:12-74 -- same kwargs; ``with_cp`` is accepted and ignored (inference path)."""

    def __init__(self, in_channels, num_stage=4, block_numbers=[2, 2, 2, 2], block_inplanes=[64, 128, 256, 512],
                 block_strides=[1, 2, 2, 2], out_indices=(0, 1, 2, 3), norm_cfg=dict(type="BN3d", requires_grad=True),
                 with_cp=True, **kwargs):
        super().__init__()
        self.out_indices = out_indices
        self.num_layers = 0
        self.layers = nn.ModuleList()
        for i in range(num_stage):
            blocks = []
            stride = block_strides[i]
            for _ in range(block_numbers[i]):
                blocks.append(DualpathTransformerBlock(in_channels, block_inplanes[i], stride=stride, norm_cfg=norm_cfg,
                                                       layer_index=self.num_layers, stage_index=i, **kwargs))
                in_channels = block_inplanes[i]
                stride = 1
                self.num_layers += 1
            self.layers.append(nn.Sequential(*blocks))
        self.with_cp = with_cp

    @torch.no_grad()
    def forward_cl(self, x_cl, x_s=None):
        """-> list of (fp32, S32) channel-last pairs, one per out_indices stage."""
        res = []
        for index, layer in enumerate(self.layers):
            for bi, blk in enumerate(layer):
                wanted = index in self.out_indices and bi == len(layer) - 1
                x_cl, x_s = blk.forward_cl(x_cl, x_s, want_f32=wanted)
            if index in self.out_indices:
                res.append((x_cl, x_s))
        return res

    def forward(self, x):
        return [to_reference_layout(f, t) for f, t in self.forward_cl(*to_channel_last(x))]
