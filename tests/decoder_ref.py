"""fp64 restatement of the decoder layer's query-side kernels, one launch at a time, in plain torch (any device).

The functions take the values a kernel is given (fp32 tensors, weights in the K-major (in, out) layout of
head._prepare()) in fp64 and return what that launch computes.  tests/test_gpu_decoder_layer.py compares the kernels with
them; tests/test_cpu_decoder_reference.py checks them against oracle.port, so a GPU failure points at the kernel."""
import torch
import torch.nn.functional as F

KEYS_PER_TILE = 128  # keys per tile of occ_cross_attn_tc
MAX_CHUNKS = 96      # key chunks (partials) per (sample, head) at most
HEAD_DIM = 32
LN_EPS = 1e-5


def chunking(S):
    """(tiles per chunk, chunks) of occ_cross_attn_tc for S keys: chunk c holds keys [c * tpc * 128, (c + 1) * tpc * 128)"""
    tiles = -(-S // KEYS_PER_TILE)
    tpc = -(-tiles // MAX_CHUNKS)
    return tpc, -(-tiles // tpc)


def encode_ordered(x):
    """fp32 pooled mask logits -> the kernels' order-preserving int32 codes: the float bits for x >= 0, bits ^ 0x7FFFFFFF
    below, -0.0 -> 0 (as +0.0).  Blocked (sigmoid(x) < 0.5) <=> code < 0."""
    i = x.float().contiguous().view(torch.int32)
    code = torch.where(i >= 0, i, i ^ 0x7FFFFFFF)
    return torch.where(i == -2 ** 31, torch.zeros_like(code), code)


def mask_words(blocked, S):
    """blocked (B, S, Q) bool -> the (B, 4 * ceil(S / 128), Q) int32 words of occ_mask_bits: bit k of word w is set iff key
    32 w + k is blocked or >= S"""
    B, _, Q = blocked.shape
    NW = 4 * -(-S // KEYS_PER_TILE)
    full = torch.ones((B, NW * 32, Q), dtype=torch.int64, device=blocked.device)
    full[:, :S] = blocked.long()
    shift = torch.arange(32, device=blocked.device).view(1, 1, 32, 1)
    w = (full.view(B, NW, 32, Q) << shift).sum(2)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def _heads(x, H):
    """(B, n, E) -> (B, H, n, E / H)"""
    B, n, E = x.shape
    return x.view(B, n, H, E // H).transpose(1, 2)


def attention(q, k, v, blocked, H):
    """Masked multi-head attention of already scaled queries: q (B, Q, E), k / v (B, S, E), blocked (B, Q, S) bool
    (True = key not attended) -> (B, Q, E).  One head at a time, to bound the (B, Q, S) score tensor."""
    out = torch.empty_like(q)
    hd = q.shape[-1] // H
    for h in range(H):
        cols = slice(h * hd, (h + 1) * hd)
        s = (q[..., cols] @ k[..., cols].transpose(1, 2)).masked_fill(blocked, float("-inf"))
        out[..., cols] = s.softmax(-1) @ v[..., cols]
    return out


def partials(q, k, v, blocked, H):
    """The key-chunk partials of occ_cross_attn_tc: (B, H, nchunk, Q, 2 + hd) = (m, l, acc) per chunk with m = max score
    of the un-blocked keys, l = sum exp(s - m), acc = sum exp(s - m) v; a chunk without an un-blocked key is (-inf, 0, 0)."""
    B, Q, E = q.shape
    S = k.shape[1]
    hd = E // H
    tpc, nchunk = chunking(S)
    part = q.new_zeros((B, H, nchunk, Q, 2 + hd))
    for h in range(H):
        cols = slice(h * hd, (h + 1) * hd)
        for c in range(nchunk):
            keys = slice(c * tpc * KEYS_PER_TILE, min(S, (c + 1) * tpc * KEYS_PER_TILE))
            s = (q[..., cols] @ k[:, keys, cols].transpose(1, 2)).masked_fill(blocked[..., keys], float("-inf"))
            m = s.amax(-1)
            p = (s - torch.where(torch.isinf(m), torch.zeros_like(m), m)[..., None]).exp()
            part[:, h, c, :, 0] = m
            part[:, h, c, :, 1] = p.sum(-1)
            part[:, h, c, :, 2:] = p @ v[:, keys, cols]
    return part


def merge(part):
    """partials (B, H, nchunk, Q, 2 + hd) -> attention output (B, Q, H * hd): every chunk rescaled to the common maximum"""
    B, H, _, Q, w = part.shape
    m = part[..., 0]
    M = m.amax(2, keepdim=True)
    scale = torch.where(torch.isinf(m), torch.zeros_like(m), (m - M).exp())
    L = (part[..., 1] * scale).sum(2)
    A = (part[..., 2:] * scale[..., None]).sum(2)
    return (A / L[..., None]).permute(0, 2, 1, 3).reshape(B, Q, H * (w - 2))


def layer_norm(x, w, b):
    return F.layer_norm(x, (x.shape[-1],), w, b, LN_EPS)


def cross_merge(att, query, qpos, L, scale):
    """occ_cross_merge after the partial merge: att / query / qpos (rows, E) -> (query1, sa_qkv (rows, 3E)).
    query1 = LN(norms.0)(att Wo^T + bo + query); sa_qkv = self-attention in-projection [q * scale | k | v] with
    q, k from query1 + qpos and v from query1."""
    E = query.shape[-1]
    q1 = layer_norm(att @ L["ca_woT"] + L["ca_bo"] + query, L["n0w"], L["n0b"])
    p = q1 + qpos
    W, b = L["sa_inT"], L["sa_inb"]
    sa = torch.cat([(p @ W[:, :E] + b[:E]) * scale, p @ W[:, E:2 * E] + b[E:2 * E], q1 @ W[:, 2 * E:] + b[2 * E:]], 1)
    return q1, sa


def self_attn_ffn(sa, q1, Qs, nkeys, L, H):
    """occ_self_attn_ffn: every query slot of a sample attends to the first nkeys slots -> (x1, y) with
    x1 = LN(norms.1)(attention Wo^T + bo + query1) and y = x1 + FFN(x1), the input of the closing LN(norms.2)."""
    rows, E = q1.shape
    B = rows // Qs
    qkv = sa.view(B, Qs, 3 * E)
    k, v = qkv[:, :nkeys, E:2 * E], qkv[:, :nkeys, 2 * E:]
    blocked = torch.zeros((B, Qs, nkeys), dtype=torch.bool, device=sa.device)
    att = attention(qkv[..., :E].contiguous(), k.contiguous(), v.contiguous(), blocked, H).reshape(rows, E)
    x1 = layer_norm(att @ L["sa_woT"] + L["sa_bo"] + q1, L["n1w"], L["n1b"])
    y = x1 + F.relu(x1 @ L["f1T"] + L["f1b"]) @ L["f2T"] + L["f2b"]
    return x1, y


def query_head(query_in, W, norm2=None, next_q=None):
    """occ_query_head -> (query, cls, membed, qh): query = LN(norm2)(query_in) when norm2 = (w, b), else query_in;
    post_norm -> cls_embed and the 3-layer mask-embed MLP; next_q = (qpos rows, wqT, bq, scale) adds the next layer's
    cross-attention query projection qh = ((query + qpos) Wq^T + bq) * scale."""
    q = layer_norm(query_in, *norm2) if norm2 is not None else query_in
    qh = None
    if next_q is not None:
        qpos, wqT, bq, scale = next_q
        qh = ((q + qpos) @ wqT + bq) * scale
    x = layer_norm(q, W["pn_w"], W["pn_b"])
    cls = x @ W["clsT"] + W["cls_b"]
    m = F.relu(x @ W["m0T"] + W["m0b"])
    m = F.relu(m @ W["m1T"] + W["m1b"])
    return q, cls, m @ W["m2T"] + W["m2b"], qh


def prepared_weights(sd, layer=0):
    """(head, layer) weight dicts of a head state dict in the layout of head._prepare() (K-major (in, out) matrices),
    for an embedding width no head can be built with: the sine positional encoding needs E % 3 == 0, the kernels take
    E = 256.  tests/test_cpu_decoder_reference.py checks that this equals _prepare() where a head can be built."""
    T = lambda w: w.detach().float().t().contiguous()  # noqa: E731
    V = lambda w: w.detach().float().contiguous()      # noqa: E731
    E = sd["transformer_decoder.post_norm.weight"].numel()
    W = dict(pn_w=V(sd["transformer_decoder.post_norm.weight"]), pn_b=V(sd["transformer_decoder.post_norm.bias"]),
             clsT=T(sd["cls_embed.weight"]), cls_b=V(sd["cls_embed.bias"]))
    for i, n in ((0, "m0"), (2, "m1"), (4, "m2")):
        W[n + "T"], W[n + "b"] = T(sd[f"mask_embed.{i}.weight"]), V(sd[f"mask_embed.{i}.bias"])
    p = f"transformer_decoder.layers.{layer}."
    ca, sa = p + "attentions.0.attn.", p + "attentions.1.attn."
    L = dict(ca_wqT=T(sd[ca + "in_proj_weight"][:E]), ca_bq=V(sd[ca + "in_proj_bias"][:E]),
             ca_woT=T(sd[ca + "out_proj.weight"]), ca_bo=V(sd[ca + "out_proj.bias"]),
             sa_inT=T(sd[sa + "in_proj_weight"]), sa_inb=V(sd[sa + "in_proj_bias"]),
             sa_woT=T(sd[sa + "out_proj.weight"]), sa_bo=V(sd[sa + "out_proj.bias"]),
             f1T=T(sd[p + "ffns.0.layers.0.0.weight"]), f1b=V(sd[p + "ffns.0.layers.0.0.bias"]),
             f2T=T(sd[p + "ffns.0.layers.1.weight"]), f2b=V(sd[p + "ffns.0.layers.1.bias"]))
    for n in range(3):
        L[f"n{n}w"], L[f"n{n}b"] = V(sd[p + f"norms.{n}.weight"]), V(sd[p + f"norms.{n}.bias"])
    return W, L


def to64(d, device=None):
    """dict of fp32 tensors (a layer or the head of head._prepare()) -> fp64 copies"""
    return {k: v.detach().to(device=device, dtype=torch.float64) for k, v in d.items() if torch.is_tensor(v)}
