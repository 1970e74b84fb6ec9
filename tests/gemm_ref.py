"""fp64 restatement of the split-bf16 GEMM / implicit-GEMM conv (csrc/gemm_bf16x3.cu: occ_gemm_bf16x3, occ_conv_bf16x3,
occ_conv_slice_bf16x3, occ_conv_taps_bf16x3) and of the host's tile dispatch, plus the case table of
tests/test_gpu_gemm_instances.py.

Every contraction returns two fp64 results of the same inputs:
  true      the exact product of the fp32 operands (fp64 products of fp32 values are exact);
  emulated  what the kernel's passes compute when every product and sum is exact: the operands split bit for bit as
            ops.split_weight does (hi = bf16(x), lo = bf16(x - hi)), then sum hi.hi' + lo.hi' + hi.lo' (three passes) or
            sum hi.hi' (the single-pass bf16 mode).  The lo.lo' term is the one the three passes leave out.
The epilogue follows the kernel's order: bias, then residual, then the activation (ReLU, GELU(erf), Swish), in fp64.
The GroupNorm statistics are fp64 (sum, sumsq) per (sample, group) of the raw (pre-epilogue) output.

Gates (tests/util.assert_close, both criteria):
  GATE          kernel vs true fp64.  The three passes leave out lo.lo' (<= 2^-18 of each product) and round hi and lo.
  emu_gate()    kernel vs the emulation: what remains is wgmma's fp32 accumulation and the fp32 epilogue.  The tensor
                core does not round its fp32 accumulation to nearest: every wgmma shrinks the partial sums by up to about
                2^-24 of their size, so the difference grows with the number of wgmmas that accumulate into an output
                (2 * passes per k-block) and is nearly a uniform scale (rel_rms close to rel_max).  Measured on one NVIDIA
                H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock) over the 470 launches of the case table, the
                least tolerance passing both criteria was at most 2.1 x 2^-24 per wgmma (7.4e-7 at one k-block, 3.8e-5 at
                81 k-blocks of 256-row tiles); the single-pass mode, at most 1.6 x 2^-24 per wgmma (2.1e-6 at 216
                k-blocks).  The gate is (16 + 6 * passes * k-blocks) * 2^-24: 3 x 2^-24 per wgmma, plus 16 ulps for
                the epilogue -- 2.3x to 3.6x the measured figures at every depth.  Below about 15 k-blocks it is tighter
                than GATE, so a mistake GATE would dilute (one border row, one partial column) stands out; deeper, GATE
                is the tighter of the two.
  stats_gate()  the GroupNorm statistics vs those of the emulated output: (16 + 2 * passes * k-blocks) * 2^-24 (measured
                at most 0.43 x 2^-24 per wgmma: 1.25e-5 at 81 k-blocks; the sums of squares shrink twice as fast).

The `mistake` arguments plant the mistakes a kernel change is likely to make; tests/test_cpu_gemm_reference.py checks,
on the GPU test's own inputs, that each moves the emulated result by more than 10 x the case's emu_gate() (a k-block's
hi.lo' or lo.hi' term, about 2^-10 of that block, by more than 2 x: at depth the truncation above is within 10x of
it).  They exist for that check only."""
import math

import torch
import torch.nn.functional as F

from encoder_ref import case_seed  # one seed rule for every kernel-level test

GATE = 5e-5


def emu_gate(nkb, passes=3):
    """kernel vs emulation for a contraction of nkb 32-k blocks (see above)"""
    return (16 + 6 * passes * nkb) * 2.0 ** -24


def stats_gate(nkb, passes=3):
    return (16 + 2 * passes * nkb) * 2.0 ** -24


SMS = 132            # the H100 SXM's SM count: the tile counts and conv plans below assume it
BM, BK = 128, 32
MAX_STAT_GROUPS = 96
PLANT = 4.0          # the last k-block of every weight is scaled by this (see weights())

KBLOCK_MISTAKES = ("hi*lo' dropped in the last k-block", "lo*hi' dropped in the last k-block")
EPILOGUE_MISTAKES = ("bias after the activation", "residual after the activation", "last row dropped",
                     "last partial column dropped")
TAP_MISTAKES = tuple(f"last tap along {a} read one voxel off" for a in "xyz")
STATS_MISTAKES = ("group statistics credited to the next group",)


# ------------------------------------------------------------------------------------------------ operands
def split(x):
    """fp32 tensor -> (hi, lo) fp64, bit for bit as ops.split_weight: hi = bf16(x), lo = bf16(x - hi)"""
    x = x.float()
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi.double(), lo.double()


def _kblock_cols(K, splits, kb_per_tap=None):
    """the k-blocks the k-block mistakes drop: the last one of each split, as (block, tap, block in tap)"""
    nkb = K // BK
    out = []
    for s in range(splits):
        kb = (s + 1) * nkb // splits - 1
        out.append((kb,) + ((kb // kb_per_tap, kb % kb_per_tap) if kb_per_tap else (0, kb)))
    return out


def contract(a, w, passes=3, mistake=None):
    """plain GEMM a (M, K) @ w (N, K)^T of fp32 operands -> (true, emulated), fp64 (M, N), on a's device"""
    true = a.double() @ w.double().t()
    ah, al = split(a)
    wh, wl = split(w)
    emu = ah @ (wh + wl).t() + al @ wh.t() if passes == 3 else ah @ wh.t()
    if mistake in KBLOCK_MISTAKES:
        for kb, _, _ in _kblock_cols(a.shape[1], 1):
            c = slice(kb * BK, (kb + 1) * BK)
            emu = emu - (ah[:, c] @ wl[:, c].t() if mistake.startswith("hi*lo'") else al[:, c] @ wh[:, c].t())
    elif mistake is not None:
        raise ValueError(mistake)
    return true, emu


def epilogue(y, bias=None, residual=None, act=0, mistake=None):
    """the kernel's epilogue on a raw fp64 result y (rows, N): + bias, + residual, then act (0 none, 1 ReLU, 2 GELU(erf),
    3 Swish).  Mistakes: bias / residual added after the activation, the last row or the last column of a partial
    32-column chunk left at zero."""
    f = [lambda v: v, torch.relu, F.gelu, lambda v: v * torch.sigmoid(v)][act]
    b = None if bias is None else bias.double()
    r = None if residual is None else residual.double().reshape(y.shape)
    late_b = mistake == "bias after the activation"
    late_r = mistake == "residual after the activation"
    if b is not None and not late_b:
        y = y + b
    if r is not None and not late_r:
        y = y + r
    y = f(y)
    if b is not None and late_b:
        y = y + b
    if r is not None and late_r:
        y = y + r
    if mistake == "last row dropped":
        y = y.clone()
        y[-1] = 0
    elif mistake == "last partial column dropped":
        assert y.shape[1] % 32, "no partial chunk"
        y = y.clone()
        y[:, -1] = 0
    elif mistake not in (None, "bias after the activation", "residual after the activation"):
        raise ValueError(mistake)
    return y


def gemm_ref(a, w, bias=None, residual=None, act=0, passes=3, mistake=None):
    """occ_gemm_bf16x3 -> (true, emulated) fp64 (M, N)"""
    kb = mistake if mistake in KBLOCK_MISTAKES else None
    true, emu = contract(a, w, passes, kb)
    return epilogue(true, bias, residual, act), epilogue(emu, bias, residual, act, None if kb else mistake)


def gn_stats(y, B, cpg, mistake=None):
    """fp64 (sum, sumsq) per (sample, group) of y (B * rows, C) -> (B, C / cpg, 2).  Mistake: group 0's sums added to
    group 1's and group 0 left at zero."""
    v = y.double().reshape(B, -1, y.shape[-1] // cpg, cpg)
    s = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1)
    if mistake == STATS_MISTAKES[0]:
        assert s.shape[1] >= 2, "one group only"
        s = s.clone()
        s[:, 1] += s[:, 0]
        s[:, 0] = 0
    elif mistake is not None:
        raise ValueError(mistake)
    return s


# ------------------------------------------------------------------------------------------------ convolution
def out_size(n, k, stride, dil):
    p = dil * (k - 1) // 2
    return (n + 2 * p - dil * (k - 1) - 1) // stride + 1


def stencil_taps(k, dil):
    """the input offsets (padding folded in) of a regular KX x KY x KZ stencil, in the kernel's tap order (x-major)"""
    pads = [dil * (kk - 1) // 2 for kk in k]
    return [(i * dil - pads[0], j * dil - pads[1], l * dil - pads[2])
            for i in range(k[0]) for j in range(k[1]) for l in range(k[2])]


def _range(n_out, n_in, s, off):
    """outputs o with 0 <= o * s + off < n_in -> (output slice, input slice)"""
    lo = max(0, (-off + s - 1) // s)
    hi = min(n_out, (n_in - 1 - off) // s + 1)
    if hi <= lo:
        return None
    return slice(lo, hi), slice(lo * s + off, (hi - 1) * s + off + 1, s)


def tap_sum(x, w, taps, stride, out_shape):
    """sum over taps t of x shifted by taps[t] (zero outside the grid) times w[:, t]^T: x (B, X, Y, Z, Cin),
    w (Cout, T, Cin), output (B, Xo, Yo, Zo, Cout), all fp64; output voxel o reads input o * stride + offset"""
    B, X, Y, Z, _ = x.shape
    Xo, Yo, Zo = out_shape
    out = torch.zeros(B, Xo, Yo, Zo, w.shape[0], dtype=torch.float64, device=x.device)
    for t, (ox, oy, oz) in enumerate(taps):
        r = [_range(Xo, X, stride, ox), _range(Yo, Y, stride, oy), _range(Zo, Z, stride, oz)]
        if None in r:
            continue
        (xo, xi), (yo, yi), (zo, zi) = r
        out[:, xo, yo, zo] += x[:, xi, yi, zi] @ w[:, t].t()
    return out


def _conv3d(x, w, stride, dil):
    """x (B, X, Y, Z, Cin), w (Cout, Cin, KX, KY, KZ) fp64 -> "same"-padded F.conv3d, channel-last"""
    pad = tuple(dil * (kk - 1) // 2 for kk in w.shape[2:])
    return F.conv3d(x.permute(0, 4, 1, 2, 3), w, None, stride, pad, dil).permute(0, 2, 3, 4, 1)


def conv_contract(x, w, stride=1, dil=1, passes=3, splits=1, mistake=None):
    """occ_conv_bf16x3's raw output: x (B, X, Y, Z, Cin), w (Cout, Cin, KX, KY, KZ) fp32 -> (true, emulated) fp64
    (B, Xo, Yo, Zo, Cout), three (or two, by linearity) fp64 F.conv3d calls.  `splits` = the plan's K splits (where the
    k-block mistakes drop their block)."""
    true = _conv3d(x.double(), w.double(), stride, dil)
    xh, xl = split(x)
    wh, wl = split(w)
    emu = _conv3d(xh, wh + wl, stride, dil) + _conv3d(xl, wh, stride, dil) if passes == 3 else _conv3d(xh, wh, stride, dil)
    if mistake is not None:
        emu = emu + conv_mistake(x, w, stride, dil, passes, splits, mistake)
    return true, emu


def conv_mistake(x, w, stride, dil, passes, splits, mistake):
    """what a planted mistake adds to conv_contract's emulated output (by shifted sums over the taps it concerns)"""
    xh, xl = split(x)
    wh, wl = split(w)
    k = tuple(w.shape[2:])
    taps = stencil_taps(k, dil)
    Cout, Cin = w.shape[:2]
    tw = lambda t: t.permute(0, 2, 3, 4, 1).reshape(Cout, len(taps), Cin)  # noqa: E731 -- tap-major, as repacked
    shape = tuple(out_size(n, kk, stride, dil) for n, kk in zip(x.shape[1:4], k))
    delta = torch.zeros(x.shape[0], *shape, Cout, dtype=torch.float64, device=x.device)
    if mistake in KBLOCK_MISTAKES:
        a, b = (xh, tw(wl)) if mistake.startswith("hi*lo'") else (xl, tw(wh))
        for _, t, cb in _kblock_cols(len(taps) * Cin, splits, Cin // BK):
            c = slice(cb * BK, (cb + 1) * BK)
            delta -= tap_sum(a[..., c], b[:, t:t + 1, c], [taps[t]], stride, shape)
    elif mistake in TAP_MISTAKES:
        ax = "xyz".index(mistake.split()[3])
        idx = [(i, j, l) for i in range(k[0]) for j in range(k[1]) for l in range(k[2])]
        pairs = [(xh, tw(wh + wl)), (xl, tw(wh))] if passes == 3 else [(xh, tw(wh))]
        for t in (t for t, i in enumerate(idx) if i[ax] == k[ax] - 1):
            off = list(taps[t])
            off[ax] += 1
            for a, b in pairs:
                delta += tap_sum(a, b[:, t:t + 1], [tuple(off)], stride, shape) - tap_sum(a, b[:, t:t + 1], [taps[t]],
                                                                                          stride, shape)
    else:
        raise ValueError(mistake)
    return delta


def taps_contract(x, w2, taps, passes=3, mistake=None):
    """occ_conv_taps_bf16x3's raw output: x (B, X, Y, Z, Cin), w2 (Cout, ntaps * Cin) fp32 tap-major, taps [(dx, dy, dz)]
    -> (true, emulated) fp64 (B, X, Y, Z, Cout), by explicit shifted sums.  Mistake: the last tap read one voxel off
    along x."""
    Cout, Cin = w2.shape[0], x.shape[-1]
    w = w2.reshape(Cout, len(taps), Cin)
    shape = tuple(x.shape[1:4])
    true = tap_sum(x.double(), w.double(), taps, 1, shape)
    xh, xl = split(x)
    wh, wl = split(w)
    read = list(taps)
    if mistake == TAP_MISTAKES[0]:
        read[-1] = (read[-1][0] + 1,) + tuple(read[-1][1:])
    elif mistake is not None:
        raise ValueError(mistake)
    emu = tap_sum(xh, wh + wl, read, 1, shape) + tap_sum(xl, wh, read, 1, shape) if passes == 3 \
        else tap_sum(xh, wh, read, 1, shape)
    return true, emu


def conv_ref(x, w, stride=1, dil=1, bias=None, residual=None, act=0, passes=3, cpg=0, splits=1, taps=None,
             mistake=None):
    """occ_conv_bf16x3 / occ_conv_slice_bf16x3 (w (Cout, Cin, KX, KY, KZ)) or, with taps, occ_conv_taps_bf16x3
    (w (Cout, ntaps * Cin)) -> (true, emulated, true stats, emulated stats); outputs (B, Xo, Yo, Zo, Cout) fp64, stats
    of the raw output (B, Cout / cpg, 2) or None without cpg"""
    cm = mistake if mistake in KBLOCK_MISTAKES + TAP_MISTAKES else None
    sm = mistake if mistake in STATS_MISTAKES else None
    em = None if cm or sm else mistake
    if taps is None:
        true, emu = conv_contract(x, w, stride, dil, passes, splits, cm)
    else:
        true, emu = taps_contract(x, w, taps, passes, cm)
    B, Cout = true.shape[0], true.shape[-1]
    st = se = None
    if cpg:
        st, se = gn_stats(true.reshape(B, -1, Cout), B, cpg), gn_stats(emu.reshape(B, -1, Cout), B, cpg, sm)
    shp = true.shape
    ep = lambda y, m=None: epilogue(y.reshape(-1, Cout), bias, residual, act, m).view(shp)  # noqa: E731
    return ep(true), ep(emu, em), st, se


# ------------------------------------------------------------------------------------------------ tile dispatch
def gemm_bn(N):
    return 32 if N <= 32 else 64 if N <= 64 else 96 if (N % 96 == 0 and N % 128 != 0) else 128


def gemm_stages(bn, mt):
    return 4 if mt == 2 else 8 if bn <= 32 else 6 if bn <= 64 else 4 if bn <= 96 else 3


def conv_box(Xo, Yo, Zo, rows, stride):
    padded = lambda n, b: (n + b - 1) // b * b  # noqa: E731
    best, box = -1, None
    z = rows
    while z >= 1:
        y = rows // z
        while y >= 1:
            x = rows // (z * y)
            if not (x * stride > 256 or y * stride > 256 or z * stride > 256):
                v = padded(Xo, x) * padded(Yo, y) * padded(Zo, z)
                if best < 0 or v < best:
                    best, box = v, (x, y, z)
            y >>= 1
        z >>= 1
    return box


def conv_plan(B, Xo, Yo, Zo, Cout, stride, nkb, splitk_ok, sms=SMS):
    """occ_conv_bf16x3's tiling -> dict(mt, bn, stages, splits, box, tiles (x, y, z), m_tiles)"""
    bn = gemm_bn(Cout)
    n_tiles = (Cout + bn - 1) // bn

    def tile(rows):
        box = conv_box(Xo, Yo, Zo, rows, stride)
        t = tuple((n + b - 1) // b for n, b in zip((Xo, Yo, Zo), box))
        return box, t, B * t[0] * t[1] * t[2]

    mt, splits = 1, 1
    box2, t2, m2 = tile(2 * BM)
    box1, t1, m1 = tile(BM)
    if bn in (96, 128) and nkb >= 64 and m2 * n_tiles >= 4 * sms and m2 * 2 * 100 <= m1 * 105:
        mt, box, t, m = 2, box2, t2, m2
    else:
        box, t, m = box1, t1, m1
        tiles = m1 * n_tiles

        def eff(s):
            tt = tiles * s
            return tt / (((tt + sms - 1) // sms) * sms)

        if splitk_ok and m1 >= 8 and tiles < 2 * sms and nkb >= 64 and eff(1) < 0.85:
            best = 1
            for sp in range(2, 9):
                if sp * 8 > nkb:
                    break
                if eff(sp) > eff(best) + 0.02:
                    best = sp
                if eff(best) >= 0.85:
                    break
            splits = best
    return dict(mt=mt, bn=bn, stages=gemm_stages(bn, mt), splits=splits, box=box, tiles=t, m_tiles=m,
                n_tiles=n_tiles)


def label(mt, bn, lean, tma, split):
    """an instantiation gemm_bf16x3_kernel<BN, STAGES, LEAN, MT> and the store path of a launch"""
    kind = "lean" if lean else "MT2" if mt == 2 else "full"
    return f"{kind} BN{bn} {'TMA' if tma else 'scalar'}{' split-K' if split else ''}"


# every instantiation x {TMA store, scalar stores where reachable} x {split-K where reachable}.  LEAN needs the TMA store
# and one split; split-K needs the TMA store and 128-row tiles.
REQUIRED = ({label(1, bn, True, True, False) for bn in (64, 96, 128)}
            | {label(1, bn, False, tma, sp) for bn in (32, 64, 96, 128) for tma, sp in ((True, False), (False, False),
                                                                                         (True, True))}
            | {label(2, bn, False, tma, False) for bn in (96, 128) for tma in (True, False)})


# ------------------------------------------------------------------------------------------------ the case table
# Plain GEMM: name -> (M, N, K, bias, residual, act, split_out, bias_misaligned, out_misaligned)
def G(M, N, K, bias=False, residual=False, act=0, split_out=False, mis_bias=False, mis_out=False):
    return dict(M=M, N=N, K=K, bias=bias, residual=residual, act=act, split_out=split_out, mis_bias=mis_bias,
                mis_out=mis_out)


def gemm_label(c):
    N = c["N"]
    tma = N % 4 == 0 and not c["mis_out"]
    bn = gemm_bn(N)
    lean = tma and N % 32 == 0 and not c["mis_bias"] and bn != 32
    return label(1, bn, lean, tma, False)


def gemm_tiles(c):
    return (c["M"] + BM - 1) // BM * ((c["N"] + gemm_bn(c["N"]) - 1) // gemm_bn(c["N"]))


GEMM_BIG = {  # more tiles than SMs: every CTA runs the persistent loop at least twice
    "lean BN64": G(40000, 64, 96),                  # 3 k-blocks in a 6-deep ring
    "lean BN96": G(20000, 192, 160),                # 5 k-blocks in a 4-deep ring
    "lean BN128": G(17000, 256, 32),                # 1 k-block: the ring phase wraps inside a tile boundary
    "full BN32": G(17000, 32, 64, bias=True),
    "full BN64": G(17000, 48, 64, bias=True),       # partial chunk
    "full BN96": G(9000, 192, 96, bias=True, mis_bias=True),
    "full BN128": G(17100, 100, 64, residual=True),  # partial chunk
    "scalar BN32": G(17100, 18, 64, bias=True),
    "scalar BN32 N6": G(3000, 6, 32),
    "scalar BN64": G(17100, 50, 64, residual=True),
    "scalar BN96 misaligned out": G(17100, 96, 64, bias=True),
    "scalar BN128": G(17100, 126, 96, bias=True),
}
GEMM_BIG["scalar BN96 misaligned out"]["mis_out"] = True

# M at the tile edges, on a lean, a full-epilogue (partial chunk) and a scalar-store shape
GEMM_EDGES = {f"M{M} N{N}": G(M, N, 64, bias=True) for M in (1, 127, 128, 129, 257) for N in (64, 100, 18)}

# act 0-3 x bias x residual on every plain-GEMM instantiation and store path (M = 300: three M tiles); the bases below
# reach their instantiation whatever bias / residual they get: a misaligned bias keeps BN 96 / 128 off the lean path,
# a misaligned output sends BN 96 to the scalar stores
EPI_BASES = {
    "lean BN64": G(300, 64, 96), "lean BN96": G(300, 192, 160), "lean BN128": G(300, 256, 32),
    "full BN32": G(300, 32, 64), "full BN64": G(300, 48, 64), "full BN96": G(300, 192, 96, mis_bias=True),
    "full BN128": G(300, 100, 64), "scalar BN32": G(300, 18, 64), "scalar BN64": G(300, 50, 64),
    "scalar BN96": G(300, 96, 64, mis_out=True), "scalar BN128": G(300, 126, 64),
}
GEMM_EPI = {}
for _n, _b in EPI_BASES.items():
    for _act in range(4):
        for _bias in (False, True):
            for _res in (False, True):
                if _b["mis_bias"] and not _bias:
                    continue  # without a bias there is nothing to misalign: that launch is the lean one
                GEMM_EPI[f"{_n} act{_act} bias{int(_bias)} res{int(_res)}"] = dict(_b, bias=_bias, residual=_res, act=_act)
# split_out at every BN with N % 32 == 0 (bias misaligned on BN 128 to reach the full epilogue)
GEMM_SPLIT_OUT = {
    "lean BN64": G(300, 64, 96, bias=True, act=1, split_out=True),
    "lean BN96": G(300, 192, 160, bias=True, act=2, split_out=True),
    "lean BN128": G(300, 256, 32, residual=True, act=3, split_out=True),
    "full BN32": G(300, 32, 64, bias=True, residual=True, act=1, split_out=True),
    "full BN96": G(300, 192, 96, bias=True, mis_bias=True, act=2, split_out=True),
    "full BN128": G(300, 256, 64, bias=True, mis_bias=True, residual=True, act=3, split_out=True),
}
GEMM_CASES = {**{f"big {k}": v for k, v in GEMM_BIG.items()}, **{f"edge {k}": v for k, v in GEMM_EDGES.items()},
              **{f"epi {k}": v for k, v in GEMM_EPI.items()}, **{f"split_out {k}": v for k, v in GEMM_SPLIT_OUT.items()}}


def gemm_inputs(c):
    """fp32 (a (M, K), w (N, K), bias (N,) or None, residual (M, N) or None) of a plain-GEMM case"""
    M, N, K = c["M"], c["N"], c["K"]
    g = torch.Generator().manual_seed(case_seed(M, N, K))
    a = torch.randn(M, K, generator=g)
    w = weights(torch.randn(N, K, generator=g) * K ** -0.5)
    bias = torch.randn(N, generator=g) if c["bias"] else None
    res = torch.randn(M, N, generator=g) if c["residual"] else None
    return a, w, bias, res


def weights(w2):
    """a weight matrix (N, K) in the kernel's k order with its last k-block scaled by PLANT: that block's hi.lo' and
    lo.hi' terms then stand out of the rest of the sum"""
    w2 = w2.clone()
    w2[:, -BK:] *= PLANT
    return w2


# Conv contractions (the inputs every conv case of the same base shares): name -> (B, X, Y, Z, Cin, Cout, k, stride, dil)
CONV_BASES = {
    "k133 B3": (3, 24, 20, 12, 32, 32, (1, 3, 3), 1, 1),       # BN 32, more tiles than SMs across 3 samples
    "k313": (2, 13, 11, 9, 32, 48, (3, 1, 3), 1, 1),           # BN 64, partial chunk
    "k331": (1, 17, 15, 6, 64, 96, (3, 3, 1), 1, 1),           # BN 96
    "s2 odd": (2, 15, 13, 9, 32, 128, (3, 3, 3), 2, 1),        # BN 128, stride 2 on odd sizes
    "dil2": (1, 14, 12, 10, 32, 60, (3, 3, 3), 1, 2),          # BN 64, dilation 2 on all three axes, Cout 60
    "tiny": (1, 1, 9, 1, 32, 64, (3, 3, 3), 1, 1),             # X = 1, Z = 1 with KZ = 3: smaller than one voxel box
    "odd Cout": (1, 12, 10, 8, 32, 126, (3, 3, 3), 1, 1),      # BN 128, Cout % 4 != 0: scalar stores
    "Cout18": (2, 9, 8, 7, 32, 18, (3, 3, 3), 1, 1),           # BN 32 scalar stores
    "Cout50": (1, 10, 9, 8, 64, 50, (3, 1, 3), 1, 1),          # BN 64 scalar stores
    "Cout192": (1, 20, 20, 4, 64, 192, (3, 3, 3), 1, 1),       # BN 96, up to 96 groups
    # 256-row tiles: Cout 192 (BN 96) and its first 128 / 126 output channels (BN 128, TMA / scalar stores)
    "MT2": (1, 64, 60, 36, 96, 192, (3, 3, 3), 1, 1),
    # split-K (no epilogue, contiguous output, a workspace)
    "splitK BN32": (1, 16, 16, 8, 96, 32, (3, 3, 3), 1, 1),
    "splitK BN64": (1, 16, 16, 8, 96, 60, (3, 3, 3), 1, 1),
    "splitK BN96": (1, 20, 20, 4, 256, 96, (3, 3, 3), 1, 1),
    "splitK BN128": (1, 25, 25, 4, 128, 128, (3, 3, 3), 1, 1),
    "splitK z-wrap": (1, 23, 28, 8, 96, 128, (3, 3, 3), 1, 1),  # three splits: they start at taps 9 and 18, block 0
}
MT2_COLS = {"MT2 BN96": 192, "MT2 BN128": 128, "MT2 BN128 scalar": 126}


def conv_inputs(base):
    """fp32 (x (B, X, Y, Z, Cin), w (Cout, Cin, KX, KY, KZ)) of a conv base; the weights' last k-block (last tap, last
    32 input channels) scaled by PLANT"""
    B, X, Y, Z, Cin, Cout, k, stride, dil = CONV_BASES[base]
    g = torch.Generator().manual_seed(case_seed(B, X, Y, Z, Cin, Cout, *k, stride, dil))
    x = torch.randn(B, X, Y, Z, Cin, generator=g)
    w = torch.randn(Cout, Cin, *k, generator=g) * (Cin * math.prod(k)) ** -0.5
    w[:, -BK:, k[0] - 1, k[1] - 1, k[2] - 1] *= PLANT
    return x, w


def conv_nkb(base):
    B, X, Y, Z, Cin, Cout, k, stride, dil = CONV_BASES[base]
    return math.prod(k) * Cin // BK


def conv_out_shape(base):
    B, X, Y, Z, Cin, Cout, k, stride, dil = CONV_BASES[base]
    return tuple(out_size(n, kk, stride, dil) for n, kk in zip((X, Y, Z), k))


# conv launches: name -> dict(base, cols (the first Cout output channels of the base), cpg, bias, residual, act,
# split_out, out ("contig", "misaligned": 4 bytes past a 16-byte boundary, "slice": columns [off, off + Cout) of an
# ldo-wide sentinel buffer), ldo, off, splitk (a workspace is passed: the launch may split K))
def C(base, cols=None, cpg=0, bias=False, residual=False, act=0, split_out=False, out="contig", ldo=0, off=0,
      splitk=False):
    return dict(base=base, cols=cols or CONV_BASES[base][5], cpg=cpg, bias=bias, residual=residual, act=act,
                split_out=split_out, out=out, ldo=ldo, off=off, splitk=splitk)


CONV_CASES = {
    "k133 B3 cpg1": C("k133 B3", cpg=1),
    "k133 B3 epi": C("k133 B3", bias=True, residual=True, act=3),
    "k313 cpg16": C("k313", cpg=16),
    "k313 epi": C("k313", bias=True, act=2),
    "k331 cpg3": C("k331", cpg=3),
    "k331 cpg12": C("k331", cpg=12),
    "k331 cpg24": C("k331", cpg=24),
    "k331 cpg48": C("k331", cpg=48),
    "k331 cpg96": C("k331", cpg=96),
    "k331 scalar": C("k331", bias=True, act=1, out="misaligned"),
    "s2 odd cpg64": C("s2 odd", cpg=64),
    "s2 odd epi": C("s2 odd", bias=True, residual=True, act=1),
    "dil2 cpg5": C("dil2", cpg=5),
    "tiny": C("tiny", cpg=8, bias=True, act=2),
    "odd Cout": C("odd Cout", cpg=6, bias=True, residual=True),
    "Cout18": C("Cout18", cpg=9, bias=True, act=3),
    "Cout50": C("Cout50", cpg=5, residual=True, act=1),
    "Cout192 cpg2": C("Cout192", cpg=2),
    "Cout192 cpg6": C("Cout192", cpg=6),
    "MT2 BN96 cpg6": C("MT2", cpg=6),
    "MT2 BN96 cpg2": C("MT2", cpg=2),
    "MT2 BN96 gelu": C("MT2", bias=True, act=2),
    "MT2 BN96 res split_out": C("MT2", residual=True, split_out=True, act=1),
    "MT2 BN96 scalar": C("MT2", bias=True, out="misaligned"),
    "MT2 BN96 slice fp32": C("MT2", bias=True, act=1, out="slice", ldo=264, off=36),
    "MT2 BN96 slice s32": C("MT2", bias=True, split_out=True, out="slice", ldo=288, off=64),
    "MT2 BN128 swish": C("MT2", 128, bias=True, residual=True, act=3),
    "MT2 BN128 cpg64": C("MT2", 128, cpg=64),
    "MT2 BN128 scalar": C("MT2", 126, cpg=42, bias=True, act=1),
    "k331 slice fp32": C("k331", act=1, bias=True, out="slice", ldo=108, off=8),
    "k331 slice s32": C("k331", split_out=True, out="slice", ldo=160, off=32),
    "splitK BN32": C("splitK BN32", cpg=8, splitk=True),
    "splitK BN64": C("splitK BN64", cpg=5, splitk=True),
    "splitK BN96": C("splitK BN96", cpg=48, splitk=True),
    "splitK BN128": C("splitK BN128", cpg=4, splitk=True),
    "splitK z-wrap": C("splitK z-wrap", cpg=64, splitk=True),
}


def conv_case_plan(c):
    """the plan the launch of conv case c takes, from the dispatch rules"""
    B, X, Y, Z, Cin, _, k, stride, dil = CONV_BASES[c["base"]]
    Cout = c["cols"]
    Xo, Yo, Zo = conv_out_shape(c["base"])
    ldo = c["ldo"] or Cout
    tma = Cout % 4 == 0 and ldo % 4 == 0 and c["out"] != "misaligned"
    splitk_ok = (tma and ldo == Cout and not (c["bias"] or c["residual"] or c["act"] or c["split_out"])
                 and c["splitk"])
    return conv_plan(B, Xo, Yo, Zo, Cout, stride, math.prod(k) * Cin // BK, splitk_ok), tma, splitk_ok


def conv_label(c):
    plan, tma, _ = conv_case_plan(c)
    return label(plan["mt"], plan["bn"], False, tma, plan["splits"] > 1)


def split_boundaries(c):
    """(tap, block in tap) at which each split but the first starts (split-K cases)"""
    B, X, Y, Z, Cin, _, k, stride, dil = CONV_BASES[c["base"]]
    nkb, cb = math.prod(k) * Cin // BK, Cin // BK
    s = conv_case_plan(c)[0]["splits"]
    return [((i * nkb // s) // cb, (i * nkb // s) % cb) for i in range(1, s)]


# tap tables: name -> (B, X, Y, Z, Cin, Cout, taps, cpg)
TAP_CASES = {
    "3-D offsets": (2, 9, 7, 6, 32, 64, [(0, 0, 0), (-1, 2, -3), (3, -2, 1), (-4, -1, 2), (1, 1, -1), (2, 0, 4),
                                         (100, 0, 0), (-2, -5, 0)], 16),
    "one tap": (1, 12, 10, 5, 64, 32, [(1, -1, 2)], 4),
    "28 taps": (1, 10, 9, 6, 32, 96, [(0, -127, 127)] + [(i % 3 - 1, (i // 3) % 3 - 1, i // 9 - 1) for i in range(27)],
                24),
}


def taps_inputs(name):
    B, X, Y, Z, Cin, Cout, taps, _ = TAP_CASES[name]
    g = torch.Generator().manual_seed(case_seed(B, X, Y, Z, Cin, Cout, len(taps)))
    x = torch.randn(B, X, Y, Z, Cin, generator=g)
    w2 = weights(torch.randn(Cout, len(taps) * Cin, generator=g) * (len(taps) * Cin) ** -0.5)
    return x, w2


def tap_label(name):
    B, X, Y, Z, Cin, Cout, taps, _ = TAP_CASES[name]
    return label(1, gemm_bn(Cout), False, True, False)


def epilogue_inputs(rows, N, c):
    """fp32 (bias (N,) or None, residual (rows, N) or None) of a conv case"""
    g = torch.Generator().manual_seed(case_seed(rows, N, c["act"], c["bias"], c["residual"]))
    bias = torch.randn(N, generator=g) if c["bias"] else None
    res = torch.randn(rows, N, generator=g) if c["residual"] else None
    return bias, res
