"""Inference-time weight folding (float64 on the host, stored fp32 on the device).

* Conv(no bias)+BatchNorm(eval) -> one affine map                 (reference encoder_utils.py:28-34)
* P_out_proj + P_integration (two cat + 1x1 Conv+BN with no activation in between,
  reference deepinteraction_encoder.py:13-14,26-27) -> ONE linear map over [a | b | c]
* single-head MMRI_I2P attention: K/V projections folded into the query / output side
  (SURVEY.md section 0 item 1; reference encoder_utils.py:223-224,311-318)
"""
import math

import torch


ON_DEVICE = [False]     # train.py: fold on the parameters' device (no host round trip, hence no stream synchronisation)


def _d(t):
    t = t.detach().double()
    return t if ON_DEVICE[0] else t.cpu()


class on_device:
    """Context: the folding helpers of this module keep their float64 intermediates on the parameters' device."""

    def __enter__(self):
        self.saved, ON_DEVICE[0] = ON_DEVICE[0], True

    def __exit__(self, *a):
        ON_DEVICE[0] = self.saved


def conv_bn(conv, bn=None):
    """-> (W [Cout, Cin*k*k] float64 in torch layout order, b [Cout])."""
    W = _d(conv.weight)
    b = _d(conv.bias) if conv.bias is not None else torch.zeros(W.shape[0], dtype=torch.float64)
    if bn is not None:
        g = _d(bn.weight) if bn.weight is not None else torch.ones_like(b)
        beta = _d(bn.bias) if bn.bias is not None else torch.zeros_like(b)
        s = g / torch.sqrt(_d(bn.running_var) + bn.eps)
        W = W * s.view(-1, *([1] * (W.dim() - 1)))
        b = (b - _d(bn.running_mean)) * s + beta
    return W, b


def pointwise(cb):
    """ConvBN holder (1x1) -> (W [Cout,Cin], b)."""
    W, b = conv_bn(cb.conv, getattr(cb, 'bn', None))
    return W.reshape(W.shape[0], -1), b


def pack_conv3x3(W):
    """[Cout,Cin,3,3] -> [Cout, (ky*3+kx)*Cin + ci]"""
    return W.permute(0, 2, 3, 1).reshape(W.shape[0], -1)


def fuse_pair(out_proj, integration):
    """new = integration(cat(out_proj(cat(a, b)), c))  ->  Wf [C, 3C], bf with new = Wf @ [a;b;c] + bf."""
    W1, b1 = pointwise(out_proj)          # [C, 2C]
    W2, b2 = pointwise(integration)       # [C, 2C]
    C = W1.shape[0]
    W2a, W2b = W2[:, :C], W2[:, C:]
    return torch.cat([W2a @ W1, W2b], 1), W2a @ b1 + b2


def i2p_fold(mha, split_bias=False):
    """nn.MultiheadAttention (1 head) -> M1 [Ck, Cq], c1, M2 [Cq, Ck], c2 with
    qk = M1 q + c1;  out = M2 (sum_j a_j k_j) + c2.
    split_bias (attention dropout, weights a_j m_j that no longer sum to 1): -> M1, c1, M2x [Cq, Ck + 4], b_o with
    out = M2x [s, rho, 0, 0, 0] + b_o, s = sum_j a_j m_j k_j, rho = sum_j a_j m_j, M2x = [W_o W_v | W_o b_v | 0 0 0]."""
    E = mha.embed_dim
    assert mha.num_heads == 1
    if mha._qkv_same_embed_dim:
        Wq, Wk, Wv = _d(mha.in_proj_weight).chunk(3, 0)
    else:
        Wq, Wk, Wv = _d(mha.q_proj_weight), _d(mha.k_proj_weight), _d(mha.v_proj_weight)
    bq, bk, bv = _d(mha.in_proj_bias).chunk(3, 0)
    Wo, bo = _d(mha.out_proj.weight), _d(mha.out_proj.bias)
    s = 1.0 / math.sqrt(E)
    M1 = Wk.T @ Wq * s
    c1 = Wk.T @ bq * s
    M2 = Wo @ Wv
    if split_bias:
        return M1, c1, torch.cat([M2, (Wo @ bv)[:, None], torch.zeros_like(M2[:, :3])], 1), bo
    c2 = Wo @ bv + bo
    return M1, c1, M2, c2


def i2p_unfold_grads(mha, dM1, dc1, dM2, dc2):
    """Chain rule of i2p_fold: gradients w.r.t. the folded (M1, c1, M2, c2) -> gradients of the attention module's own
    parameters, float64 on the host: dict(Wq, Wk, Wv, bq, bk, bv, Wo, bo).  (bk does not influence the output: it adds
    the same constant to every logit of a pillar.)"""
    E = mha.embed_dim
    if mha._qkv_same_embed_dim:
        Wq, Wk, Wv = _d(mha.in_proj_weight).chunk(3, 0)
    else:
        Wq, Wk, Wv = _d(mha.q_proj_weight), _d(mha.k_proj_weight), _d(mha.v_proj_weight)
    bq, bk, bv = _d(mha.in_proj_bias).chunk(3, 0)
    Wo = _d(mha.out_proj.weight)
    s = 1.0 / math.sqrt(E)
    dM1, dc1, dM2, dc2 = (_d(t) for t in (dM1, dc1, dM2, dc2))
    dbo = dc2
    Ck = Wv.shape[1]
    if dM2.shape[1] == Ck + 4:                 # i2p_fold(split_bias=True): column Ck is d(W_o b_v), dc2 is d b_o alone
        dM2, dc2 = dM2[:, :Ck], dM2[:, Ck]
    # M1 = s Wk^T Wq, c1 = s Wk^T bq, M2 = Wo Wv, c2 = Wo bv + bo
    return dict(Wq=s * Wk @ dM1, bq=s * Wk @ dc1, Wk=s * (Wq @ dM1.T + torch.outer(bq, dc1)), bk=torch.zeros_like(bk),
                Wv=Wo.T @ dM2, Wo=dM2 @ Wv.T + torch.outer(dc2, bv), bv=Wo.T @ dc2, bo=dbo)


def decoder_layer_unfold_consts(layer, num_heads, device, dtype=torch.float32):
    """Constants of decoder_layer_unfold for one TransformerDecoderLayer (built once per pack): the q-row scale of the
    in-projections and, per positional MLP, the first convolution's weight and bias minus the BN running mean, the BN
    1 / sqrt(var + eps) and gamma."""
    C = layer.self_attn.embed_dim
    s = float(C // num_heads) ** -0.5
    u = dict(C=C, s=s, qscale=torch.cat([torch.full((C,), s, dtype=torch.float64), torch.ones(2 * C, dtype=torch.float64)]))
    for name in ('self_posembed', 'cross_posembed'):
        seq = getattr(layer, name).position_embedding_head
        u[name] = conv_bn_unfold_consts(seq[0], seq[1])
    cast = lambda t: t.to(device=device, dtype=dtype) if torch.is_tensor(t) else t
    return {k: (tuple(cast(x) for x in v) if isinstance(v, tuple) else cast(v)) for k, v in u.items()}


def conv_bn_unfold_consts(conv, bn):
    """Constants of conv_bn_unfold for one convolution + BatchNorm (eval) pair, float64 on the host: the convolution's weight
    as [Cout, Cin*k*k], its bias (0 without one) minus the BN running mean, the BN 1 / sqrt(var + eps) and gamma."""
    W0 = _d(conv.weight).reshape(conv.weight.shape[0], -1)
    b0 = _d(conv.bias) if conv.bias is not None else torch.zeros(W0.shape[0], dtype=torch.float64)
    return W0, b0 - _d(bn.running_mean), 1.0 / torch.sqrt(_d(bn.running_var) + bn.eps), _d(bn.weight)


def conv_bn_unfold(consts, dW1, db1):
    """Chain rule of the conv + BN fold W1 = W0 sc, b1 = (b0 - mean) sc + beta, sc = gamma / sqrt(var + eps), from the
    gradients of the folded (W1 [Cout, Cin*k*k], b1) -> (d W0, d b0, d gamma, d beta).  consts: conv_bn_unfold_consts
    (cast where the gradients are)."""
    W0, b0m, inv, gamma = consts
    sc = gamma * inv
    return dW1 * sc[:, None], db1 * sc, ((dW1 * W0).sum(1) + db1 * b0m) * inv, db1


def decoder_layer_unfold(u, g):
    """Chain rule from the gradients of the packed, folded weights of the decoder layer (mmpi pack: 'self_attn',
    'cross_q', 'cross_kv', 'self_pe', 'cross_pe') to the parameters of the TransformerDecoderLayer, keyed and shaped as
    in its state_dict.  u: decoder_layer_unfold_consts.  Runs where the tensors are (no host round trip).
    g: self_in (dW [3C, 2C] of [W_s | W_s] over [query | query_pos_embed], db [3C]), cross_q (dW [C, 2C] of [Wq_s | Wq_s],
    db [C]), cross_kv (dW [2C, C], db [2C]), self_posembed / cross_posembed (dW1 [C, cin], db1 of the conv + BN fold, dW2
    [C, C], db2).  W_s has its q rows scaled by head_dim^-0.5 (s); the BN fold is W1 = W0 sc, b1 = (b0 - mean) sc + beta,
    sc = gamma / sqrt(var + eps)."""
    C, s = u['C'], u['s']
    out = {}
    dWp, db = g['self_in']
    out['self_attn.in_proj_weight'] = (dWp[:, :C] + dWp[:, C:]) * u['qscale'][:, None]
    out['self_attn.in_proj_bias'] = db * u['qscale']
    dWq, dbq = g['cross_q']
    dWkv, dbkv = g['cross_kv']
    out['multihead_attn.in_proj_weight'] = torch.cat([(dWq[:, :C] + dWq[:, C:]) * s, dWkv], 0)
    out['multihead_attn.in_proj_bias'] = torch.cat([dbq * s, dbkv])
    for name in ('self_posembed', 'cross_posembed'):
        dW1, db1, dW2, db2 = g[name]
        pre = name + '.position_embedding_head.'
        dW0, db0, dgamma, dbeta = conv_bn_unfold(u[name], dW1, db1)
        out[pre + '0.weight'] = dW0.unsqueeze(-1)
        out[pre + '0.bias'] = db0
        out[pre + '1.weight'] = dgamma
        out[pre + '1.bias'] = dbeta
        out[pre + '3.weight'] = dW2.unsqueeze(-1)
        out[pre + '3.bias'] = db2
    return out


def dev(t, device):
    return t.to(torch.float32).contiguous().to(device)


def split_tf32(w):
    """fp32 tensor -> (hi, lo): hi = w rounded (nearest-even) to TF32's 10 mantissa bits, lo = w - hi (exact)."""
    w = w.to(torch.float32).contiguous()
    bits = w.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    rounded = (bits + 0x0FFF + ((bits >> 13) & 1)) & 0xFFFFE000
    hi = (rounded & 0xFFFFFFFF).to(torch.int64)
    hi = torch.where(hi >= 2 ** 31, hi - 2 ** 32, hi).to(torch.int32).view(torch.float32)
    return hi.contiguous(), (w - hi).contiguous()


def split_bf16(w):
    """fp32 tensor -> (hi, mid) bf16: hi = bf16(w), mid = bf16(w - hi); hi + mid keeps 16 mantissa bits of w."""
    w = w.to(torch.float32).contiguous()
    hi = w.to(torch.bfloat16)
    mid = (w - hi.to(torch.float32)).to(torch.bfloat16)
    return hi.contiguous(), mid.contiguous()


def split_rows(x, kind):
    """Host model of the pre-split operand format of the window kernel (gemm_tc.cu epilogue): x [M, C] fp32 ->
    [M, C] fp32-typed tensor whose 32-bit words are packed bf16x2 (hi = bf16(x), mid = bf16(x - hi), lower channel in
    the low half).  kind 1: channel pair j -> words 2j (hi), 2j+1 (mid); kind 2: channel group of 8 -> 4 hi | 4 mid;
    kind 3 (planar window kernel): channel group of 128 -> 64 hi words | 64 mid words."""
    x = x.to(torch.float32)
    hi = x.to(torch.bfloat16)
    mid = (x - hi.to(torch.float32)).to(torch.bfloat16)
    bits = lambda t: t.view(torch.int16).to(torch.int32) & 0xFFFF
    pack = lambda b: (b[:, 0::2] | (b[:, 1::2] << 16))                  # [M, C/2] words
    wh, wm = pack(bits(hi)), pack(bits(mid))
    M, C = x.shape
    out = torch.empty(M, C, dtype=torch.int32, device=x.device)
    if kind == 1:
        out[:, 0::2], out[:, 1::2] = wh, wm
    elif kind == 3:
        assert C % 128 == 0
        o = out.view(M, C // 128, 128)
        o[:, :, :64], o[:, :, 64:] = wh.view(M, C // 128, 64), wm.view(M, C // 128, 64)
    else:
        o = out.view(M, C // 8, 8)
        o[:, :, :4], o[:, :, 4:] = wh.view(M, C // 8, 4), wm.view(M, C // 8, 4)
    return out.view(torch.float32)


class Weight:
    """A dense-layer weight [N, K] kept in the forms the kernels consume: plain fp32 (FFMA path), the TF32 hi/lo
    split and the bf16 hi/mid split (tensor-core paths)."""

    def __init__(self, w, device, lazy=False):
        """lazy: build the two splits on first use (training: weights change every step and only one split is read)."""
        self.w = dev(w, device)
        self.shape = self.w.shape
        self._wt = self._tf32 = self._bf16 = None
        if not lazy:
            self._tf32 = tuple(t.to(device) for t in split_tf32(w.to(torch.float32)))
            self._bf16 = tuple(t.to(device) for t in split_bf16(w))

    def _get_tf32(self):
        if self._tf32 is None:
            self._tf32 = split_tf32(self.w)
        return self._tf32

    def _get_bf16(self):
        if self._bf16 is None:
            self._bf16 = split_bf16(self.w)
        return self._bf16

    hi = property(lambda self: self._get_tf32()[0])
    lo = property(lambda self: self._get_tf32()[1])
    bh = property(lambda self: self._get_bf16()[0])
    bm = property(lambda self: self._get_bf16()[1])

    @property
    def wt(self):
        """fp32 weight transposed to [K, N] (input channel major) for the query-row MLP kernel (di_rows_mlp_f32)."""
        if self._wt is None:
            self._wt = self.w.t().contiguous()
        return self._wt
