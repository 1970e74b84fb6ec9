"""Per-kernel timings at BASELINE sizes (CUDA events, L2 flushed between iterations).  Development aid;
bench.py is the contract benchmark.  usage: python scripts/microbench.py [conv convs gemm attn tail neck lift]"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from occformer_b200 import ops, synth

dev = torch.device("cuda:0")
flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1.0)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    res = {}
    which = sys.argv[1:] or ["conv", "gemm", "attn", "tail", "neck", "lift"]
    X, Y, Z, C = 200, 200, 16, 128
    rows = X * Y * (Z + 1)
    if "conv" in which:
        x = torch.randn(1, X, Y, Z, C, device=dev)
        xs = ops.to_split(x)
        w = torch.randn(C, C, 3, 3, 3) * 0.02
        w2, ks = ops.repack_conv_weight(w)
        w2 = w2.to(dev)
        stats = torch.zeros(1, 32, 2, dtype=torch.float64, device=dev)
        t = timeit(lambda: ops.conv(xs, w2, ks, gn_stats=stats, cpg=4))
        fl = 2 * 27 * C * C * X * Y * Z
        res["conv3d_c128_bf16x3_ms"] = t
        res["conv3d_c128_alg_TFs"] = fl / t / 1e9
        # library context: cuDNN channels-last-3d, TF32 (1 pass, ~4e-4 error) and strict fp32
        xc = x.permute(0, 4, 1, 2, 3).contiguous(memory_format=torch.channels_last_3d)
        wc = w.to(dev).contiguous(memory_format=torch.channels_last_3d)
        for name, flag in (("tf32", True), ("fp32", False)):
            torch.backends.cudnn.allow_tf32 = flag
            torch.backends.cudnn.benchmark = True
            try:
                res[f"cudnn_conv3d_{name}_ms(context)"] = timeit(lambda: torch.nn.functional.conv3d(xc, wc, padding=1), iters=3)
            except Exception as e:  # noqa: BLE001
                res[f"cudnn_conv3d_{name}_ms(context)"] = str(e)[:80]
        # neck output conv 192 -> 192
        E = 192
        xe = ops.to_split(torch.randn(1, X, Y, Z, E, device=dev))
        we, ke = ops.repack_conv_weight(torch.randn(E, E, 3, 3, 3) * 0.02)
        we = we.to(dev)
        t = timeit(lambda: ops.conv(xe, we, ke), iters=3)
        res["conv3d_c192_bf16x3_ms"] = t
        res["conv3d_c192_alg_TFs"] = 2 * 27 * E * E * X * Y * Z / t / 1e9
        del x, xs, xc, xe
    if "convs" in which:
        # every 3x3x3 conv shape of one bench step (batch 4, nusc_200 grid, GroupNorm statistics as the pipeline asks
        # for them), in three passes and in one: a one-pass time close to the three-pass time means the kernel is bound by
        # operand bytes or latency, not by the tensor pipe.  Ceiling = H100 SXM data-sheet dense bf16 (989 TF/s) / 3.
        Bc = 4
        shapes = [  # name, Cin, Cout, input grid, stride, cpg
            ("c128_s1_200x200x16", 128, 128, (200, 200, 16), 1, 4),
            ("c192_s1_200x200x16", 192, 192, (200, 200, 16), 1, 6),
            ("c128to256_s2_to100x100x8", 128, 256, (200, 200, 16), 2, 8),
            ("c256_s1_100x100x8", 256, 256, (100, 100, 8), 1, 8),
            ("c256to512_s2_to50x50x4", 256, 512, (100, 100, 8), 2, 16),
            ("c512_s1_50x50x4", 512, 512, (50, 50, 4), 1, 16),
            ("c512to1024_s2_to25x25x2", 512, 1024, (50, 50, 4), 2, 32),
            ("c1024_s1_25x25x2", 1024, 1024, (25, 25, 2), 1, 32),
        ]
        for name, ci, co, (xi, yi, zi), s, cpg in shapes:
            xs = ops.to_split(torch.randn(Bc, xi, yi, zi, ci, device=dev) * 0.5)
            w2, ks = ops.repack_conv_weight(torch.randn(co, ci, 3, 3, 3) * 0.02)
            w2 = w2.to(dev)
            st = torch.zeros(Bc, co // cpg, 2, dtype=torch.float64, device=dev)
            vout = Bc * ((xi - 1) // s + 1) * ((yi - 1) // s + 1) * ((zi - 1) // s + 1)
            fl = 2.0 * 27 * ci * co * vout
            for mode in ("fp32", "bf16"):
                with ops.precision(mode):
                    t = timeit(lambda: ops.conv(xs, w2, ks, stride=s, gn_stats=st, cpg=cpg), iters=5)
                tfs = fl / t / 1e9
                res[f"{name}_{mode}"] = {"ms": round(t, 3), "alg_TFs": round(tfs, 1),
                                         "frac_of_3pass_ceiling": round(3 * tfs / 989.0, 3)}
            del xs
    if "gemm" in which:
        a = ops.to_split(torch.randn(rows, C, device=dev))
        w = ops.split_weight(torch.randn(3 * C, C) * C ** -0.5).to(dev)
        b = torch.randn(3 * C, device=dev)
        res["gemm_qkv_split_out_ms"] = timeit(lambda: ops.gemm(a, w, bias=b, split_out=True))
        a2 = ops.to_split(torch.randn(91250, 192, device=dev))
        w2 = ops.split_weight(torch.randn(768, 192) * 192 ** -0.5).to(dev)
        res["gemm_neck_ffn1_91250x768x192_ms"] = timeit(lambda: ops.gemm(a2, w2, act=1, split_out=True))
        del a, a2
    if "attn" in which:
        heads = C // 32
        tokn = ops.to_split(torch.randn(rows, C, device=dev))
        wq = ops.split_weight(torch.randn(3 * C, C) * C ** -0.5).to(dev)
        bq = torch.randn(3 * C, device=dev) * 0.1
        bqs = ops.split_weight(bq.cpu().view(1, -1)).view(-1).to(dev)
        bias_pad = torch.randn(heads, 2404, device=dev) * 0.1
        qkv = ops.gemm(tokn, wq, bias=bq, split_out=True)
        res["window_attn_tc_ms"] = timeit(lambda: ops.window_attention(qkv, bqs, bias_pad, 1, X, Y, Z, C, heads, True, head_major=True))
        tokn_wl = ops.to_window_layout(tokn, 1, X, Y, Z, True)
        res["swin_qkv_attn_fused_ms"] = timeit(lambda: ops.swin_qkv_attention(tokn_wl, wq, bq, bias_pad, 1, X, Y, Z, C, heads, True))
        tokn_wl0 = ops.to_window_layout(tokn, 1, X, Y, Z, False)
        res["swin_qkv_attn_fused_unshifted_ms"] = timeit(lambda: ops.swin_qkv_attention(tokn_wl0, wq, bq, bias_pad, 1, X, Y, Z, C, heads, False))
        del tokn_wl, tokn_wl0
        del qkv, tokn
    if "tail" in which:
        M = rows
        att = ops.to_split(torch.randn(M, C, device=dev))
        tok = torch.randn(M, C, device=dev)
        ws = [ops.split_weight(torch.randn(C, C) * C ** -0.5).to(dev) for _ in range(3)]
        bs = [torch.randn(C, device=dev) * 0.1 for _ in range(3)]
        lw, lb = torch.ones(C, device=dev), torch.zeros(C, device=dev)
        res["swin_mlp_fused_ms"] = timeit(lambda: ops.swin_proj_ffn(att, tok, ws[0], bs[0], lw, lb, ws[1], bs[1], ws[2], bs[2]))
        del att, tok
    if "neck" in which:
        E, H, L, P = 192, 8, 3, 4
        grids = [(25, 25, 2), (50, 50, 4), (100, 100, 8)]
        Nq = sum(a * b * c for a, b, c in grids)
        v = torch.randn(Nq, E, device=dev)
        ow = torch.cat([torch.randn(Nq, H * L * P * 3, device=dev) * 1.5, torch.randn(Nq, H * L * P, device=dev)], 1).contiguous()
        res["ms_deform_attn_91250_ms"] = timeit(lambda: ops.ms_deform_attn(v, ow, grids, [16, 8, 4], 1, E, H, P))
        vp = torch.zeros(Nq, H, 32, device=dev)
        vp[:, :, :E // H] = v.view(Nq, H, E // H)
        vp = vp.view(Nq, H * 32)
        res["ms_deform_attn_91250_padded_heads_ms"] = timeit(lambda: ops.ms_deform_attn(vp, ow, grids, [16, 8, 4], 1, E, H, P))
        # the FFN pair of one encoder layer (192 -> 768 -> 192) as two GEMMs
        x_s = ops.to_split(v)
        w1 = ops.split_weight(torch.randn(4 * E, E) * E ** -0.5).to(dev)
        w2 = ops.split_weight(torch.randn(E, 4 * E) * (4 * E) ** -0.5).to(dev)
        b1, b2 = torch.zeros(4 * E, device=dev), torch.zeros(E, device=dev)
        # (row-chunking the pair so that the hidden tensor stays in L2 was measured slower: 0.27 / 0.32 / 0.40 ms at 3 / 5 / 8
        # chunks vs 0.20 ms -- the short-K GEMMs are bound by their per-tile prologue / epilogue, not by HBM)
        res["neck_ffn_two_gemms_ms"] = timeit(lambda: ops.gemm(ops.gemm(x_s, w1, bias=b1, act=1, split_out=True), w2, bias=b2, residual=v))
        res["neck_token_prep_ms"] = timeit(lambda: ops.neck_token_prep(v, grids, 1, ln=(torch.ones(E, device=dev), torch.zeros(E, device=dev)),
                                                                   pos=v, want_pos=True))
    if "elem" in which:
        Bc, Xc_, Yc_, Zc_ = 1, 200, 200, 16
        nv = Xc_ * Yc_ * Zc_
        xv = torch.randn(nv, 128, device=dev)
        bev = torch.randn(Xc_ * Yc_, 128, device=dev)
        ident = ops.to_split(torch.randn(nv, 128, device=dev))
        cw = torch.randn(128, device=dev) * 0.1
        res["fuse_c128_s32_only_ms"] = timeit(lambda: ops.dualpath_fuse(xv, bev, cw, 0.1, ident, Bc, Xc_ * Yc_, Zc_, 128,
                                                                        identity_split=True, want_f32=False))
        res["fuse_c128_f32_and_s32_ms"] = timeit(lambda: ops.dualpath_fuse(xv, bev, cw, 0.1, ident, Bc, Xc_ * Yc_, Zc_, 128,
                                                                           identity_split=True, want_f32=True))
        del xv, ident
        E = 192
        cur = torch.randn(1, 200, 200, 16, E, device=dev)
        coarse = torch.randn(1, 100, 100, 8, E, device=dev)
        st = ops.gn_stats(cur.view(-1, E), 1, 200 * 200 * 16, E, 32)
        gw, gb = torch.ones(E, device=dev), torch.zeros(E, device=dev)
        res["gn_upsample_add_200x200x16x192_ms"] = timeit(lambda: ops.gn_upsample_add(cur, st, gw, gb, 32, coarse))
        res["gn_stats_200x200x16x192_ms"] = timeit(lambda: ops.gn_stats(cur.view(-1, E), 1, 200 * 200 * 16, E, 32))
        del cur, coarse
    if "lift" in which:
        from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel
        gc = synth.grid_config("nusc_200")
        vt = ViewTransformerLiftSplatShootVoxel(grid_config=gc, data_config={"input_size": (256, 704)}, numC_input=64,
                                                numC_Trans=C).to(dev)
        cams = {k: v.to(dev) for k, v in synth.nusc_cameras(1, 6).items()}
        dd, feat = synth.lift_inputs(1, 6, 112, 16, 44, C)
        dd, feat = dd.to(dev), feat.to(dev)
        dx, bx, nx = vt.prepared()
        t = timeit(lambda: ops.lift_splat_fused(dd, feat, vt.frustum.data, cams["rots"], cams["trans"], cams["intrins"],
                                                cams["post_rots"], cams["post_trans"], cams["bda"], 1, 6, dx, bx, nx,
                                                vt.grid_size(), with_split=True))
        Pn = 6 * 112 * 16 * 44
        alg = Pn * 4 + 6 * 16 * 44 * C * 4 + Pn * 12 + X * Y * Z * C * 4
        res["lift_splat_fused_ms(3 launches, with S32 twin)"] = t
        res["lift_splat_fused_GBps_fused_formula"] = alg / t / 1e6
        t = timeit(lambda: ops.lift_splat_fused(dd, feat, vt.frustum.data, cams["rots"], cams["trans"], cams["intrins"],
                                                cams["post_rots"], cams["post_trans"], cams["bda"], 1, 6, dx, bx, nx,
                                                vt.grid_size(), with_split=False))
        res["lift_splat_fused_ms(no twin)"] = t
        res["lift_splat_fused_GBps_no_twin"] = alg / t / 1e6
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
