"""The decoder layer's query-side kernels one launch at a time against the fp64 reference of tests/decoder_ref.py:
occ_mask_bits (exact), occ_cross_attn_tc (key-chunk partials), occ_cross_merge, occ_self_attn_ffn, occ_query_head,
occ_classmix at 21-32 classes, and one layer composed from them against oracle.port.decoder_layer.

Gates: GATE (kernel level, per tensor, tests/util.assert_close) for the fp32-faithful three-pass mode; BF16_TOL for the
single-pass mode (tests/test_gpu_bf16_mode.py).  Planted keys (a logit about 8 above the rest) make single keys visible
above the gate: key 0, key S-1, the first key of a chunk, and the keys of sample b+1 that the last (ragged) key tile of
sample b reads.  Each planted case checks its own sensitivity: the reference with that key's mask bit flipped (or the
sample-(b+1) key taken in) must differ from the true reference by more than 10x the gate."""
import pytest
import torch
import torch.nn.functional as F

import decoder_ref as ref
from oracle import port
from occformer_b200 import synth
from util import assert_close, parity_log

pytestmark = pytest.mark.gpu

GATE = 5e-5
BF16_TOL = 3e-2
PLANT = 8.0
PC = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
SCALE = 32 ** -0.5
B = 2


def _layer(cuda, E, F_, NC, seed, Q=4):
    """(state dict, head weights, layer 0 weights, all prepared weights) of a built one-layer head: the K-major layout
    the kernels get.  E = 256 has no head (its sine positional encoding needs E % 3 == 0): the same layout by hand."""
    from occformer_b200 import head as Hm
    sd = synth.make_head_state(E, Q, NC - 1, 1, 3, ffn=F_, seed=seed)
    if E % 3:
        W, L = ref.prepared_weights(sd)
        return sd, {k: v.to(cuda) for k, v in W.items()}, {k: v.to(cuda) for k, v in L.items()}, None
    h = Hm.Mask2FormerNuscOccHead(**Hm.head_cfg(E, Q, NC - 1, 1, E // 32, PC, ffn=F_))
    h.load_state_dict(sd, strict=True)
    P = h.to(cuda).eval()._prepare()
    return sd, P["head"], P["layers"][0], P


def _rel_to(diff_max, ref_t):
    return float(diff_max) / float(ref_t.abs().max())


# ------------------------------------------------------------------------------------------------ occ_mask_bits
@pytest.mark.parametrize("S", [1, 31, 128, 129, 12289])
def test_mask_bits_exact(cuda, S):
    from occformer_b200 import ops
    for Q in (4, 128, 132, 256):
        g = torch.Generator().manual_seed(1000 * S + Q)
        x = torch.randn(B, S, Q, generator=g)
        x.view(-1)[::7] = 0.0
        x.view(-1)[3::7] = -0.0
        code = ref.encode_ordered(x)
        code.view(-1)[5::11] = -1
        code.view(-1)[6::13] = 2 ** 31 - 1
        code.view(-1)[9::17] = -2 ** 31
        NW = 4 * -(-S // 128)
        bits = torch.empty((B, NW, Q), dtype=torch.int32, device=cuda)
        ops._call("occ_mask_bits", code.to(cuda), bits, B, S, Q)
        assert torch.equal(bits.cpu(), ref.mask_words(code < 0, S)), f"mask bits S={S} Q={Q}"


# ------------------------------------------------------------------------------------------------ occ_cross_attn_tc
def _special_rows(S, Q, nchunk, tpc, plants):
    """(b, q) -> pattern of the rows with a hand-made mask; the leak rows need a sample after them (b = 0)"""
    slots = list(dict.fromkeys([Q - 1, 0, Q // 2, 1]))
    names0 = ["flag0_leak", "leak", "plant0", "only0"]
    names1 = ["chunk_blocked", "only_last", "plant_last", "plant_chunk"]
    rows = {}
    for b, names in ((0, names0), (1, names1)):
        for q, name in zip(slots, names):
            if not plants and name.startswith("plant"):
                continue
            if name == "chunk_blocked" and nchunk < 2:
                continue
            if name == "plant_chunk" and nchunk < 2:
                continue
            if name in ("plant0", "plant_last") and S < 2:
                continue
            rows[(b, q)] = name
    return rows


def _cross_case(cuda, S, Q, E, ko, vo, seed, bf16_exact=False, plants=True):
    """Inputs of one occ_cross_attn_tc launch: K / V are the column slices [ko*E, ko*E+E) / [vo*E, vo*E+E) of (B*S, 3E)
    tensors, as when layers share a level.  -> dict of the fp32 inputs, the effective mask and the planted cases."""
    H = E // 32
    ld = 3 * E
    g = torch.Generator(device=cuda).manual_seed(seed)
    if bf16_exact:  # logits about +-30; bf16-representable q, k, v: hi*hi' is exact and the lo passes multiply zeros
        a = 1.33
        q = (torch.randn(B, Q, E, generator=g, device=cuda) * a).bfloat16().float()
        kw = (torch.randn(B * S, ld, generator=g, device=cuda) * a).bfloat16().float()
        vw = torch.randn(B * S, ld, generator=g, device=cuda).bfloat16().float()
    else:
        q = torch.randn(B, Q, E, generator=g, device=cuda) * 0.25
        kw = torch.randn(B * S, ld, generator=g, device=cuda) * 0.25
        vw = torch.randn(B * S, ld, generator=g, device=cuda)
    koff, voff = ko * E, vo * E
    logit = torch.randn(B, S, Q, generator=g, device=cuda)  # pooled mask logits: blocked <=> < 0
    tpc, nchunk = ref.chunking(S)
    rows = _special_rows(S, Q, nchunk, tpc, plants)
    open_ = lambda b, qq, keys: logit[b, keys, qq].abs_()  # noqa: E731
    plant_rows = []  # (b, q, sample of the key, key, kind)
    rem = S % 128
    leak_keys = []
    if rem:  # the last key tile of sample 0 also reads keys 0 .. 127 - rem of sample 1 (rows S .. S + 127 - rem)
        leak_keys = [0, 1] if min(S, 128 - rem) >= 2 else [0]
    for (b, qq), name in rows.items():
        if name == "flag0_leak":
            logit[b, :, qq] = -logit[b, :, qq].abs() - 0.1  # blocked everywhere: flag 0, attends to all S keys
            if leak_keys:
                plant_rows.append((b, qq, b + 1, leak_keys[0], "leak"))
        elif name == "leak":
            open_(b, qq, slice(0, S))
            logit[b, ::2, qq] *= -1
            if len(leak_keys) > 1:
                plant_rows.append((b, qq, b + 1, leak_keys[1], "leak"))
        elif name == "chunk_blocked":
            logit[b, (nchunk - 1) * tpc * 128:, qq] = -logit[b, (nchunk - 1) * tpc * 128:, qq].abs() - 0.1
            open_(b, qq, slice(0, 1))
        elif name == "only0":
            logit[b, :, qq] = -logit[b, :, qq].abs() - 0.1
            open_(b, qq, slice(0, 1))
        elif name == "only_last":
            logit[b, :, qq] = -logit[b, :, qq].abs() - 0.1
            open_(b, qq, slice(S - 1, S))
        else:
            key = {"plant0": 0, "plant_last": S - 1, "plant_chunk": (nchunk // 2) * tpc * 128}[name]
            open_(b, qq, slice(key, key + 1))
            plant_rows.append((b, qq, b, key, name))
    for b, qq, bk, key, _ in plant_rows:  # k so that q . k = PLANT in every head for this query
        qh = q[b, qq].view(H, 32)
        kw[bk * S + key, koff:koff + E] = (qh * (PLANT / qh.pow(2).sum(-1, keepdim=True))).view(E)
    code = ref.encode_ordered(logit)
    blocked = (code < 0).permute(0, 2, 1)  # (B, Q, S)
    flag = (~blocked).any(-1)
    eff = blocked & flag[..., None]  # a row without an un-blocked key attends everywhere
    return dict(q=q, kw=kw, vw=vw, ld=ld, koff=koff, voff=voff, code=code.contiguous(), flag=flag, eff=eff, rows=rows,
                plants=plant_rows, H=H, S=S, Q=Q, E=E)


def _kv64(c):
    E, S = c["E"], c["S"]
    k = c["kw"][:, c["koff"]:c["koff"] + E].double().view(B, S, E)
    v = c["vw"][:, c["voff"]:c["voff"] + E].double().view(B, S, E)
    return k, v


def _run_cross(c):
    from occformer_b200 import ops
    flag = c["flag"].to(torch.int32).reshape(-1).contiguous()
    return ops.cross_attn_tc(c["q"], ops.to_split(c["kw"]), ops.to_split(c["vw"]), c["ld"], c["koff"], c["voff"],
                             c["code"], flag, B, c["S"], c["Q"], c["E"], c["H"])


def _check_partials_exact(c, part):
    """m = -inf, l = 0, acc = 0 exactly for a chunk without an un-blocked key of the row; l > 0 elsewhere"""
    S = c["S"]
    tpc, nchunk = ref.chunking(S)
    has_open = torch.stack([(~c["eff"][..., i * tpc * 128:min(S, (i + 1) * tpc * 128)]).any(-1) for i in range(nchunk)],
                           1)  # (B, nchunk, Q)
    has_open = has_open[:, None].expand(-1, c["H"], -1, -1)
    closed = part[~has_open]
    assert bool((closed[:, 0] == float("-inf")).all()), "blocked chunk: m != -inf"
    assert bool((closed[:, 1:] == 0).all()), "blocked chunk: l or acc != 0"
    assert bool((part[has_open][:, 1] > 0).all()), "open chunk: l <= 0"
    assert bool(torch.isfinite(part[has_open][:, 0]).all())
    return int((~has_open).sum())


CROSS_CASES = [  # S, Q slots, E, K column block, V column block
    (1, 4, 96, 1, 1), (1, 256, 192, 1, 1), (49, 100, 192, 1, 1), (49, 152, 256, 1, 1), (127, 128, 256, 1, 1),
    (127, 4, 192, 1, 1), (129, 132, 96, 1, 1), (129, 4, 256, 1, 1), (2500, 152, 192, 1, 1), (2500, 128, 96, 1, 2),
    (12289, 256, 256, 1, 1), (12289, 132, 192, 2, 0), (80000, 100, 192, 1, 1), (80000, 256, 96, 1, 1)]


@pytest.mark.parametrize("S,Q,E,ko,vo", CROSS_CASES)
def test_cross_attn_partials_vs_fp64(cuda, S, Q, E, ko, vo):
    c = _cross_case(cuda, S, Q, E, ko, vo, seed=S * 7 + Q + E)
    part, npart = _run_cross(c)
    from occformer_b200 import _lib
    assert npart == ref.chunking(S)[1] == _lib.lib().occ_cross_attn_tc_partials(S)
    assert part.shape == (B, c["H"], npart, Q, 34)
    nclosed = _check_partials_exact(c, part)
    k, v = _kv64(c)
    q = c["q"].double()
    want = ref.attention(q, k, v, c["eff"], c["H"])
    got = ref.merge(part.double())
    tag = f"cross_attn_tc S={S} Q={Q} E={E} koff={c['koff']} voff={c['voff']} ({nclosed} blocked chunks)"
    assert_close(got, want, GATE, tag)
    for b, qq, bk, key, kind in c["plants"]:  # the planted key moves the answer well above the gate
        eff_row = c["eff"][b:b + 1, qq:qq + 1].clone()
        kb, vb = k[b:b + 1], v[b:b + 1]
        if bk == b:
            eff_row[..., key] = ~eff_row[..., key]
        else:  # the sample-(b+1) key taken into sample b
            kb, vb = torch.cat([kb, k[bk:bk + 1, key:key + 1]], 1), torch.cat([vb, v[bk:bk + 1, key:key + 1]], 1)
            eff_row = torch.cat([eff_row, torch.zeros_like(eff_row[..., :1])], -1)
        flipped = ref.attention(q[b:b + 1, qq:qq + 1], kb, vb, eff_row, c["H"])
        sens = _rel_to((flipped - want[b:b + 1, qq:qq + 1]).abs().max(), want)
        err = _rel_to((got - want)[b, qq].abs().max(), want)
        parity_log(f"[parity] {tag} planted {kind} key {key} of sample {bk} for row ({b},{qq}): sensitivity {sens:.2e}, "
                   f"row error {err:.2e} (gate {GATE:.0e})")
        assert sens > 10 * GATE, f"planted {kind}: flipping key {key} moves the reference by only {sens:.2e}"


@pytest.mark.parametrize("S,Q,E", [(12289, 132, 192), (80000, 256, 256)])
def test_cross_attn_large_logits_exact_operands(cuda, S, Q, E):
    """logits of about +-30 (online-softmax rescaling across tiles and chunks) on bf16-representable q, k, v: the
    products are exact, so the fp64 reference is the exact answer"""
    c = _cross_case(cuda, S, Q, E, 1, 1, seed=S + Q, bf16_exact=True, plants=False)
    part, _ = _run_cross(c)
    _check_partials_exact(c, part)
    k, v = _kv64(c)
    q = c["q"].double()
    s = (q[0, :, :32] @ k[0, :, :32].t())
    parity_log(f"[parity] cross_attn_tc large logits S={S}: head-0 logit range [{float(s.min()):.1f}, {float(s.max()):.1f}]")
    assert float(s.abs().max()) > 20
    assert_close(ref.merge(part.double()), ref.attention(q, k, v, c["eff"], c["H"]), GATE,
                 f"cross_attn_tc large logits S={S} Q={Q} E={E}")


def test_cross_attn_single_pass_mode(cuda):
    """ops.set_precision("bf16"): the single-pass branch of the P V products (no P_lo pass)"""
    from occformer_b200 import ops
    c = _cross_case(cuda, 2500, 100, 192, 1, 1, seed=3)
    with ops.precision("bf16"):
        part, _ = _run_cross(c)
    assert ops.set_precision("fp32") == "fp32"
    k, v = _kv64(c)
    want = ref.attention(c["q"].double(), k, v, c["eff"], c["H"])
    e = assert_close(ref.merge(part.double()), want, BF16_TOL, "cross_attn_tc single-pass bf16 S=2500 Q=100 E=192")
    assert e > GATE, "single-pass mode not active"
    part3, _ = _run_cross(c)  # the default mode is back
    assert_close(ref.merge(part3.double()), want, GATE, "cross_attn_tc after single-pass mode")


def test_cross_attn_rejects_unaligned_slices(cuda):
    """K / V slices must start on a 32-column S32 chunk: one TMA box per (key, head) is one chunk [hi | lo]"""
    from occformer_b200 import ops
    E, S, Q = 96, 129, 4
    c = _cross_case(cuda, S, Q, E, 1, 1, seed=0, plants=False)
    flag = c["flag"].to(torch.int32).reshape(-1).contiguous()
    ks, vs = ops.to_split(c["kw"]), ops.to_split(c["vw"])
    for ld, koff, voff in [(3 * E, E + 16, E), (3 * E, E, E + 4), (3 * E, 16, 16)]:
        with pytest.raises(RuntimeError):
            ops.cross_attn_tc(c["q"], ks, vs, ld, koff, voff, c["code"], flag, B, S, Q, E, E // 32)
    wide = torch.zeros((B * S, 3 * E + 4), device=cuda)
    with pytest.raises(RuntimeError):
        ops.cross_attn_tc(c["q"], wide, wide, 3 * E + 4, 0, 0, c["code"], flag, B, S, Q, E, E // 32)


# ------------------------------------------------------------------------------------------------ occ_cross_merge
@pytest.mark.parametrize("E,Qs,nchunk", [(96, 4, 1), (192, 100, 49), (256, 132, 90)])
def test_cross_merge_vs_fp64(cuda, E, Qs, nchunk):
    from occformer_b200 import ops
    H = E // 32
    _, _, L, _ = _layer(cuda, E, 2 * E, 18, seed=E + nchunk)
    g = torch.Generator(device=cuda).manual_seed(nchunk)
    rows = B * Qs
    m = (torch.rand(B, H, nchunk, Qs, generator=g, device=cuda) * 8 - 4)
    l = torch.rand(B, H, nchunk, Qs, generator=g, device=cuda) * 50 + 0.5
    acc = l[..., None] * torch.randn(B, H, nchunk, Qs, 32, generator=g, device=cuda) * 0.5
    if nchunk > 1:  # chunks without an un-blocked key; chunk (q % nchunk) of every row stays open
        closed = torch.rand(B, H, nchunk, Qs, generator=g, device=cuda) < 0.3
        closed[..., torch.arange(Qs) % nchunk, torch.arange(Qs)] = False
        closed[0, :, :, 1] = True
        closed[0, :, nchunk - 1, 1] = False  # one row with a single open chunk, the last
        m[closed], l[closed] = float("-inf"), 0.0
        acc[closed] = 0.0
    part = torch.cat([m[..., None], l[..., None], acc], -1).contiguous()
    query = torch.randn(rows, E, generator=g, device=cuda)
    qpos = torch.randn(Qs, E, generator=g, device=cuda)
    q1, sa = ops.cross_merge(part, nchunk, H, query, qpos, Qs, L, SCALE)
    L64 = ref.to64(L)
    att = ref.merge(part.double()).reshape(rows, E)
    q1_ref, sa_ref = ref.cross_merge(att, query.double(), qpos.double().repeat(B, 1), L64, SCALE)
    tag = f"cross_merge E={E} Qs={Qs} nchunk={nchunk}"
    assert_close(q1, q1_ref, GATE, f"{tag} query1")
    for i, name in enumerate(("q", "k", "v")):
        assert_close(sa[:, i * E:(i + 1) * E], sa_ref[:, i * E:(i + 1) * E], GATE, f"{tag} sa_qkv {name}")


# ------------------------------------------------------------------------------------------------ occ_self_attn_ffn + occ_query_head
@pytest.mark.parametrize("Qs,E,fe,NC", [(4, 96, 1, 18), (128, 192, 8, 192), (132, 256, 1, 18), (152, 96, 8, 96),
                                        (256, 256, 8, 256)])
def test_self_attn_ffn_query_head_vs_fp64(cuda, Qs, E, fe, NC):
    from occformer_b200 import ops
    H = E // 32
    _, W, L, _ = _layer(cuda, E, fe * E, NC, seed=Qs + E)
    W64, L64 = ref.to64(W), ref.to64(L)
    rows = B * Qs
    g = torch.Generator(device=cuda).manual_seed(Qs)
    qpos = torch.randn(Qs, E, generator=g, device=cuda)
    for nkeys in sorted({1, Qs - 2, Qs}):
        sa = torch.randn(rows, 3 * E, generator=g, device=cuda)
        sa[:, :E] *= SCALE
        q1 = torch.randn(rows, E, generator=g, device=cuda)
        tag = f"self_attn_ffn Qs={Qs} nkeys={nkeys} E={E} F/E={fe}"
        ybuf, fp = ops.self_attn_ffn(sa, q1, Qs, L, H, nkeys=nkeys)
        assert fp.shape == (fe, rows, E)
        _, y_ref = ref.self_attn_ffn(sa.double(), q1.double(), Qs, nkeys, L64, H)
        assert_close(ybuf.double() + fp.double().sum(0), y_ref, GATE, f"{tag}: ybuf + ffn partials")
        # the closing LN(norms.2), the query head and the next layer's query projection
        nq = (qpos, Qs, L["ca_wqT"], L["ca_bq"], SCALE)
        cls, membed, query, qh = ops.query_head(ybuf, W, NC, norm2=(L["n2w"], L["n2b"]), next_q=nq, ffn_part=fp)
        q_ref, cls_ref, m_ref, qh_ref = ref.query_head(y_ref, W64, norm2=(L64["n2w"], L64["n2b"]),
                                                       next_q=(qpos.double().repeat(B, 1), L64["ca_wqT"], L64["ca_bq"],
                                                               SCALE))
        assert_close(query, q_ref, GATE, f"{tag}: layer output (norms.2)")
        assert_close(cls, cls_ref, GATE, f"{tag}: query_head cls NC={NC}")
        assert_close(ops.from_split(membed), m_ref, GATE, f"{tag}: query_head mask embedding")
        assert_close(qh, qh_ref, GATE, f"{tag}: query_head next-layer query projection")
        if nkeys < Qs:  # padded slots (>= nkeys) never act as keys: huge values there change no real slot
            sa2 = sa.clone()
            sa2.view(B, Qs, 3 * E)[:, nkeys:] = 1e4
            ybuf2, fp2 = ops.self_attn_ffn(sa2, q1, Qs, L, H, nkeys=nkeys)
            real = lambda t: t.view(-1, B, Qs, E)[:, :, :nkeys]  # noqa: E731
            assert torch.equal(real(ybuf2), real(ybuf)) and torch.equal(real(fp2), real(fp)), f"{tag}: padded slots leak"
    # query head without norm2 / next_q / FFN partials (the first forward_head of the decoder)
    x = torch.randn(rows, E, generator=g, device=cuda)
    cls, membed, query, qh = ops.query_head(x, W, NC)
    assert qh is None and query is x
    _, cls_ref, m_ref, _ = ref.query_head(x.double(), W64)
    assert_close(cls, cls_ref, GATE, f"query_head plain Qs={Qs} E={E} cls NC={NC}")
    assert_close(ops.from_split(membed), m_ref, GATE, f"query_head plain Qs={Qs} E={E} mask embedding")


# ------------------------------------------------------------------------------------------------ one layer, composed
def _pool_reference(mask_ql, B_, grid, target, Qs):
    """the reference's attention mask from query-last fp32 logits: (pooled (B, Qs, So) fp32, blocked, after the reset)"""
    X, Y, Z = grid
    pooled = F.adaptive_max_pool3d(mask_ql.cpu().permute(0, 2, 1).reshape(B_, Qs, X, Y, Z), target).flatten(2)
    blocked = pooled.sigmoid() < 0.5
    reset = blocked.clone()
    reset[torch.where(reset.sum(-1) == reset.shape[-1])] = False
    return pooled, blocked, reset


def _negzero_mask(cuda, grid, Qs, seed):
    """query-last mask logits (B, V, Qs) kept away from 0, except query 5 of sample 0: <= 0 everywhere and -0.0 in one
    cell (sigmoid(-0.0) = 0.5: that cell is not blocked, so the row keeps its mask); query 7 of sample 1 is negative
    everywhere (the all-blocked reset)"""
    X, Y, Z = grid
    g = torch.Generator().manual_seed(seed)
    m = torch.randn(B, X * Y * Z, Qs, generator=g)
    m = m + 0.05 * torch.sign(m)
    m[0, :, 5] = -m[0, :, 5].abs()
    m[0, (3 * Y + 2) * Z + 1, 5] = -0.0
    m[1, :, 7] = -m[1, :, 7].abs()
    return m.to(cuda)


def test_mask_pool_negative_zero(cuda):
    """a pooled logit of exactly -0.0 is not blocked (reference: sigmoid(-0.0) < 0.5 is False): flag and bits agree"""
    from occformer_b200 import ops
    grid, target, Qs = (20, 20, 8), (10, 10, 4), 12
    mask = _negzero_mask(cuda, grid, Qs, seed=4)
    pooled_i, flag = ops.mask_pool(mask, B, grid, target, Qs)
    pooled, blocked, reset = _pool_reference(mask, B, grid, target, Qs)
    assert bool((pooled[0, 5] <= 0).all()) and bool(torch.signbit(pooled[0, 5]).all())
    assert int((pooled[0, 5] == 0).sum()) == 1  # exactly one -0.0 cell
    assert torch.equal(pooled_i.cpu().permute(0, 2, 1) < 0, blocked), "blocked cells differ from sigmoid < 0.5"
    assert torch.equal(flag.cpu().view(B, Qs) != 0, ~(blocked.all(-1))), "row flags differ from the reference reset"
    bits = torch.empty((B, 4 * -(-pooled_i.shape[1] // 128), Qs), dtype=torch.int32, device=cuda)
    ops._call("occ_mask_bits", pooled_i, bits, B, pooled_i.shape[1], Qs)
    assert torch.equal(bits.cpu(), ref.mask_words(blocked.permute(0, 2, 1), pooled_i.shape[1]))
    dec = ops.decode_ordered(pooled_i).cpu()[0, :, 5]
    assert not bool(torch.signbit(dec[dec == 0]).any())  # the -0.0 cell decodes to +0.0


def test_decoder_layer_composed_vs_port(cuda):
    """query_head (next-layer projection) -> mask_pool -> cross_attn_tc -> cross_merge -> self_attn_ffn ->
    query_head (norms.2) on one layer vs port.decoder_layer in fp64 on the same inputs, at the kernel gate; the mask
    holds a query whose pooled logits are <= 0 with one -0.0 (must stay finite and match) and an all-blocked query"""
    from occformer_b200 import ops
    E, H, Qr, Qs, NC, F_ = 192, 6, 98, 100, 18, 1536
    sd, W, L, P = _layer(cuda, E, F_, NC, seed=11, Q=Qr)
    mgrid, kgrid = (50, 50, 8), (25, 25, 4)
    S = kgrid[0] * kgrid[1] * kgrid[2]
    g = torch.Generator().manual_seed(12)
    query = torch.zeros(B, Qs, E)
    query[:, :Qr] = torch.randn(B, Qr, E, generator=g)
    qpos = torch.zeros(Qs, E)
    qpos[:Qr] = torch.randn(Qr, E, generator=g)
    mem, pos = torch.randn(B, S, E, generator=g), torch.randn(S, E, generator=g)
    kpos = mem + pos
    query_c, qpos_c = query.reshape(B * Qs, E).to(cuda), qpos.to(cuda)
    Kp = ops.gemm(ops.to_split(kpos.reshape(B * S, E).to(cuda)), P["kw"][0], bias=P["kb"][0], split_out=True)
    Vp = ops.gemm(ops.to_split(mem.reshape(B * S, E).to(cuda)), P["vw"][0], bias=P["vb"][0], split_out=True)
    mask = _negzero_mask(cuda, mgrid, Qs, seed=13)
    _, _, _, qh = ops.query_head(query_c, W, NC, next_q=(qpos_c, Qs, L["ca_wqT"], L["ca_bq"], SCALE))
    pooled, flag = ops.mask_pool(mask, B, mgrid, kgrid, Qs)
    part, nchunk = ops.cross_attn_tc(qh, Kp, Vp, E, 0, 0, pooled, flag, B, S, Qs, E, H)
    q1, sa = ops.cross_merge(part, nchunk, H, query_c, qpos_c, Qs, L, SCALE)
    ybuf, fp = ops.self_attn_ffn(sa, q1, Qs, L, H, nkeys=Qr)
    cls, _, out, _ = ops.query_head(ybuf, W, NC, norm2=(L["n2w"], L["n2b"]), ffn_part=fp)
    out = out.view(B, Qs, E)[:, :Qr]
    assert bool(torch.isfinite(out).all()), "non-finite decoder layer output"
    # reference: the attention mask of forward_head (sigmoid < 0.5 of the fp32 pooled logits) with the all-blocked reset
    _, _, reset = _pool_reference(mask, B, mgrid, kgrid, Qs)
    attn_mask = reset[:, :Qr].repeat_interleave(H, 0)
    sd64 = {k: v.double() for k, v in sd.items()}
    sf = lambda t: t.transpose(0, 1)  # noqa: E731
    want = sf(port.decoder_layer(sf(query[:, :Qr].double()), sf(mem.double()), sf(qpos[:Qr].double().expand(B, Qr, E)),
                                 sf(pos.double().expand(B, S, E)), attn_mask, sd64, "transformer_decoder.layers.0.", H))
    assert_close(out, want, GATE, "decoder layer composed vs port.decoder_layer")
    assert_close(out[0, 5], want[0, 5], GATE, "decoder layer: the -0.0 query")
    _, cls_ref, _, _ = ref.query_head(want.reshape(-1, E), ref.to64(W, "cpu"))
    assert_close(cls.view(B, Qs, NC)[:, :Qr], cls_ref.view(B, Qr, NC), GATE, "decoder layer composed: cls")


# ------------------------------------------------------------------------------------------------ occ_classmix, 21-32 classes
@pytest.mark.parametrize("K", [21, 32])
@pytest.mark.parametrize("up", [1, 2])
def test_classmix_many_classes(cuda, K, up):
    """classmix_kernel<32> (21..32 classes): identity and x2 trilinear upsample vs port.format_results in fp64, with
    Qs > Q padded slots holding large logits that must contribute nothing; labels = argmax of the kernel's own scores"""
    from occformer_b200 import ops
    NC, Q, Qs, grid = K + 1, 98, 100, (12, 10, 6)
    out_grid = tuple(up * s for s in grid)
    g = torch.Generator().manual_seed(K * up)
    V = grid[0] * grid[1] * grid[2]
    mask = torch.randn(B, V, Qs, generator=g) * 3
    mask[..., Q:] = 50.0
    cls = torch.randn(B, Q, NC, generator=g) * 2
    out, labels = ops.classmix(mask.to(cuda), cls.to(cuda), B, grid, out_grid, Q, NC, with_labels=True)
    m = mask[..., :Q].double().permute(0, 2, 1).reshape(B, Q, *grid)
    if up != 1:
        m = F.interpolate(m, size=out_grid, mode="trilinear", align_corners=True)
    want = port.format_results(cls.double(), m)
    assert_close(out, want, GATE, f"classmix K={K} {grid}->{out_grid}")
    assert torch.equal(labels.long(), out.argmax(1)), "labels are not the argmax of the class scores"
