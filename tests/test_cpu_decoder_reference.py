"""The fp64 reference of tests/test_gpu_decoder_layer.py (tests/decoder_ref.py) against oracle.port and against itself:
the chunked partials merge to unchunked attention, the launch-by-launch pieces compose to port.decoder_layer, and the
pooled-logit encoding follows the reference's sigmoid threshold.  A GPU failure then points at a kernel, not at the
reference."""
import pytest
import torch

import decoder_ref as ref
from oracle import port
from occformer_b200 import synth

PC = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]


def _layer(E, Q, K, F, seed):
    """(state dict in fp64, head weights, layer 0 weights) of a one-layer head, read through head._prepare()"""
    from occformer_b200 import head as Hm
    sd = synth.make_head_state(E, Q, K, 1, 3, ffn=F, seed=seed)
    h = Hm.Mask2FormerNuscOccHead(**Hm.head_cfg(E, Q, K, 1, E // 32, PC, ffn=F))
    h.load_state_dict(sd, strict=True)
    P = h._prepare()
    return {k: v.double() for k, v in sd.items()}, ref.to64(P["head"]), ref.to64(P["layers"][0])


def test_prepared_weights_match_head_prepare():
    """the hand-made K-major layout (for E = 256, where no head can be built) equals head._prepare()"""
    from occformer_b200 import head as Hm
    E, Q, K, F = 96, 10, 17, 192
    sd = synth.make_head_state(E, Q, K, 1, 3, ffn=F, seed=3)
    h = Hm.Mask2FormerNuscOccHead(**Hm.head_cfg(E, Q, K, 1, E // 32, PC, ffn=F))
    h.load_state_dict(sd, strict=True)
    P = h._prepare()
    W, L = ref.prepared_weights(sd)
    assert W.keys() == P["head"].keys() and L.keys() == P["layers"][0].keys()
    for got, want in ((W, P["head"]), (L, P["layers"][0])):
        for k in want:
            assert torch.equal(got[k], want[k]) and got[k].is_contiguous(), k


def test_chunking_matches_library():
    from occformer_b200 import _lib
    assert ref.chunking(12289) == (2, 49)  # a last chunk of one tile holding one key
    assert ref.chunking(80000) == (7, 90)
    lib = _lib.lib()
    for S in [1, 49, 127, 128, 129, 2500, 12288, 12289, 32768, 80000, 96 * 128 * 3 + 1]:
        assert ref.chunking(S)[1] == lib.occ_cross_attn_tc_partials(S), S


@pytest.mark.parametrize("S", [1, 129, 12289])
def test_partial_merge_equals_unchunked_attention(S):
    g = torch.Generator().manual_seed(S)
    B, Q, E, H = 2, 6, 64, 2
    q, k, v = (torch.randn(B, n, E, generator=g, dtype=torch.float64) for n in (Q, S, S))
    blocked = torch.rand(B, Q, S, generator=g) < 0.5
    blocked[:, :, 0] = False  # every row keeps an un-blocked key
    blocked[0, 1] = True
    blocked[0, 1, S - 1] = False  # only the last key
    tpc, nchunk = ref.chunking(S)
    if nchunk > 1:
        blocked[1, 2, (nchunk - 1) * tpc * 128:] = True  # a whole chunk blocked
    part = ref.partials(q, k, v, blocked, H)
    assert part.shape == (B, H, nchunk, Q, 2 + E // H)
    torch.testing.assert_close(ref.merge(part), ref.attention(q, k, v, blocked, H), rtol=1e-12, atol=1e-12)
    if nchunk > 1:
        assert torch.isinf(part[1, :, -1, 2, 0]).all() and (part[1, :, -1, 2, 1:] == 0).all()


def test_layer_pieces_compose_to_port_decoder_layer():
    """cross attention + merge tail + self attention / FFN + closing LN == port.decoder_layer, and the query head ==
    port.forward_head, on the K-major weights of a built head"""
    E, H, Qr, Qs, S, B = 96, 3, 10, 12, 300, 2
    sd, W, L = _layer(E, Qr, 17, 192, seed=5)
    g = torch.Generator().manual_seed(1)
    query = torch.randn(B, Qs, E, generator=g, dtype=torch.float64)
    qpos = torch.randn(Qs, E, generator=g, dtype=torch.float64)
    key, kpos = (torch.randn(B, S, E, generator=g, dtype=torch.float64) for _ in range(2))
    blocked = torch.rand(B, Qr, S, generator=g) < 0.6
    blocked[0, 3] = True  # a row blocked everywhere: the reference's reset
    blocked[torch.where(blocked.sum(-1) == S)] = False
    p = "transformer_decoder.layers.0."
    sf = lambda t: t.transpose(0, 1)  # noqa: E731  (B, n, E) <-> seq-first (n, B, E)
    want = sf(port.decoder_layer(sf(query[:, :Qr]), sf(key), sf(qpos[:Qr].expand(B, Qr, E)), sf(kpos),
                                 blocked.repeat_interleave(H, 0), sd, p, H))
    # the same layer as the kernels split it
    scale = 32 ** -0.5
    _, _, _, qh = ref.query_head(query.reshape(-1, E), W, next_q=(qpos.repeat(B, 1), L["ca_wqT"], L["ca_bq"], scale))
    wk, bk = sd[p + "attentions.0.attn.in_proj_weight"][E:2 * E], sd[p + "attentions.0.attn.in_proj_bias"][E:2 * E]
    wv, bv = sd[p + "attentions.0.attn.in_proj_weight"][2 * E:], sd[p + "attentions.0.attn.in_proj_bias"][2 * E:]
    kp, vp = (key + kpos) @ wk.t() + bk, key @ wv.t() + bv
    blk = torch.zeros(B, Qs, S, dtype=torch.bool)
    blk[:, :Qr] = blocked
    att = ref.merge(ref.partials(qh.view(B, Qs, E), kp, vp, blk, H))
    q1, sa = ref.cross_merge(att.reshape(-1, E), query.reshape(-1, E), qpos.repeat(B, 1), L, scale)
    x1, y = ref.self_attn_ffn(sa, q1, Qs, Qr, L, H)
    out, cls, membed, _ = ref.query_head(y, W, norm2=(L["n2w"], L["n2b"]))
    torch.testing.assert_close(out.view(B, Qs, E)[:, :Qr], want, rtol=1e-10, atol=1e-10)
    # query head: cls and mask embedding (mask features = identity, so the einsum returns the embedding itself)
    eye = torch.eye(E, dtype=torch.float64).view(1, E, E, 1, 1).expand(B, E, E, 1, 1)
    cls_ref, m_ref, _, _ = port.forward_head(sf(want), eye, (E, 1, 1), sd, H)
    torch.testing.assert_close(cls.view(B, Qs, -1)[:, :Qr], cls_ref, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(membed.view(B, Qs, E)[:, :Qr], m_ref.view(B, Qr, E), rtol=1e-10, atol=1e-10)


def test_ordered_encoding_follows_the_sigmoid_threshold():
    from occformer_b200 import ops
    # (tiny negatives such as -1e-30 are blocked here while the reference's fp32 sigmoid rounds them to 0.5: a known,
    # tolerated difference, so they are left out of the threshold check)
    x = torch.tensor([-0.0, 0.0, -3.5, 2.0, float("-inf"), float("inf"), -1e-3, 1e-3])
    code = ref.encode_ordered(x)
    assert code[0] == 0 and code[1] == 0  # -0.0 is +0.0: sigmoid(-0.0) = 0.5 is not blocked
    assert torch.equal(code < 0, torch.sigmoid(x) < 0.5)
    assert torch.equal(ops.decode_ordered(code), x)  # +0.0 == -0.0 under equality
    assert not torch.signbit(ops.decode_ordered(code[:1])).any()
    r = torch.randn(10000, generator=torch.Generator().manual_seed(0)) * 10
    c = ref.encode_ordered(r)
    assert torch.equal(torch.argsort(c), torch.argsort(r))  # order preserving


def test_mask_words_bit_layout():
    g = torch.Generator().manual_seed(2)
    B, S, Q = 2, 129, 3
    blocked = torch.rand(B, S, Q, generator=g) < 0.5
    w = ref.mask_words(blocked, S)
    assert w.shape == (B, 8, Q) and w.dtype == torch.int32
    for b in range(B):
        for q in range(Q):
            for key in range(8 * 32):
                bit = (int(w[b, key // 32, q]) >> (key % 32)) & 1
                assert bit == (1 if key >= S else int(blocked[b, key, q])), (b, q, key)
