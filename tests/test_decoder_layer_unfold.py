"""CPU: fold.decoder_layer_unfold (the map from the gradients of the decoder layer's packed, folded weights back to the
TransformerDecoderLayer parameters, which backward.decoder_layer_backward runs on the device) against float64 autograd
through the fold formulas: the head_dim^-0.5 scale of the q rows, the [W | W] self-attention pack over
[query | query_pos_embed], the q-only cross pack, the K / V rows, and the eval-mode BN1d fold of both positional MLPs."""
import torch

from deepinteraction_b200 import fold, mmpi, synth


def _layer():
    torch.manual_seed(4)
    layer = mmpi.TransformerDecoderLayer(128, 8, 256)
    synth.randomize_norm_stats(layer, 4)
    return layer.double()


def _folded(layer, p, C, s):
    """The folded weights of DeepInteractionDecoder.pack as differentiable functions of the parameters p."""
    def scaled(w):
        return torch.cat([w[:C] * s, w[C:]], 0)
    out = {}
    Ws, bs = scaled(p['self_attn.in_proj_weight']), scaled(p['self_attn.in_proj_bias'][:, None])[:, 0]
    out['self_in'] = (torch.cat([Ws, Ws], 1), bs)
    Wx, bx = scaled(p['multihead_attn.in_proj_weight']), scaled(p['multihead_attn.in_proj_bias'][:, None])[:, 0]
    out['cross_q'] = (torch.cat([Wx[:C], Wx[:C]], 1), bx[:C])
    out['cross_kv'] = (Wx[C:], bx[C:])
    for name in ('self_posembed', 'cross_posembed'):
        pre = name + '.position_embedding_head.'
        bn = getattr(layer, name).position_embedding_head[1]
        sc = p[pre + '1.weight'] / torch.sqrt(bn.running_var + bn.eps)
        W1 = p[pre + '0.weight'][:, :, 0] * sc[:, None]
        b1 = (p[pre + '0.bias'] - bn.running_mean) * sc + p[pre + '1.bias']
        out[name] = (W1, b1, p[pre + '3.weight'][:, :, 0], p[pre + '3.bias'])
    return out


def test_decoder_layer_unfold_matches_autograd_through_the_fold():
    layer = _layer()
    C, s = 128, 16 ** -0.5
    params = {n: t.detach().clone().requires_grad_(True) for n, t in layer.named_parameters()}
    with torch.enable_grad():
        folded = _folded(layer, params, C, s)
        # the differentiable formulas are the ones pack() evaluates
        for name in ('self_posembed', 'cross_posembed'):
            seq = getattr(layer, name).position_embedding_head
            W, b = fold.conv_bn(seq[0], seq[1])
            assert torch.allclose(folded[name][0], W.reshape(C, -1), rtol=1e-14, atol=0)
            assert torch.allclose(folded[name][1], b, rtol=1e-14, atol=1e-16)
        g = torch.Generator().manual_seed(5)
        G = {k: tuple(torch.randn(t.shape, generator=g, dtype=torch.float64) for t in v) for k, v in folded.items()}
        loss = sum((t * gt).sum() for k in folded for t, gt in zip(folded[k], G[k]))
        loss.backward()
    u = fold.decoder_layer_unfold_consts(layer, 8, 'cpu', torch.float64)
    got = fold.decoder_layer_unfold(u, G)
    unfolded = {n for n in params if n.startswith(('self_attn.in_proj', 'multihead_attn.in_proj', 'self_posembed',
                                                   'cross_posembed'))}
    assert set(got) == unfolded and len(unfolded) == 16
    sd = layer.state_dict()
    for n in unfolded:
        assert got[n].shape == sd[n].shape, n
        err = float((got[n] - params[n].grad).abs().max() / params[n].grad.abs().max())
        assert err < 1e-12, (n, err)
