"""CPU: fold.conv_bn_unfold on the decoder's prediction heads (ConvBN1d, no convolution bias) and heat-map head (ConvBN2d
3x3), the map backward.pred_head_backward and backward.heatmap_head_backward run on the device, against float64 autograd
through fold.conv_bn, the formula the pack evaluates."""
import pytest
import torch

from deepinteraction_b200 import fold, mmpi, synth
from deepinteraction_b200.mmri import ConvBN


@pytest.mark.parametrize('cin,k,dims', [(128, 1, 1), (256, 1, 1), (128, 3, 2)], ids=['pred_C', 'pred_2C', 'heatmap'])
def test_conv_bn_unfold_matches_autograd_through_the_fold(cin, k, dims):
    torch.manual_seed(cin + k)
    cout = 64 if dims == 1 else 128
    cb = ConvBN(cin, cout, k, dims=dims)
    synth.randomize_norm_stats(cb, 7)
    cb = cb.double()
    assert cb.conv.bias is None
    p = {n: t.detach().clone().requires_grad_(True) for n, t in cb.named_parameters()}
    bn = cb.bn
    with torch.enable_grad():
        sc = p['bn.weight'] / torch.sqrt(bn.running_var + bn.eps)
        W = p['conv.weight'].reshape(cout, -1) * sc[:, None]
        b = -bn.running_mean * sc + p['bn.bias']
        W0, b0 = fold.conv_bn(cb.conv, cb.bn)
        assert torch.allclose(W, W0.reshape(cout, -1), rtol=1e-14, atol=0) and torch.allclose(b, b0, rtol=1e-14, atol=1e-16)
        g = torch.Generator().manual_seed(3)
        gW, gb = torch.randn(W.shape, generator=g, dtype=torch.float64), torch.randn(b.shape, generator=g, dtype=torch.float64)
        ((W * gW).sum() + (b * gb).sum()).backward()
    dW, _, dgamma, dbeta = fold.conv_bn_unfold(fold.conv_bn_unfold_consts(cb.conv, cb.bn), gW, gb)
    got = {'conv.weight': dW.view(p['conv.weight'].shape), 'bn.weight': dgamma, 'bn.bias': dbeta}
    assert set(got) == set(p)
    for n, t in got.items():
        err = float((t - p[n].grad).abs().max() / p[n].grad.abs().max())
        assert err < 1e-12, (n, err)


def test_decoder_layer_unfold_is_unchanged_by_the_shared_formula():
    """decoder_layer_unfold now calls conv_bn_unfold: the same products in the same order as its own former formula."""
    torch.manual_seed(4)
    layer = mmpi.TransformerDecoderLayer(128, 8, 256)
    synth.randomize_norm_stats(layer, 4)
    u = fold.decoder_layer_unfold_consts(layer, 8, 'cpu', torch.float32)
    g = torch.Generator().manual_seed(9)
    dW1, db1 = torch.randn(128, 2, generator=g), torch.randn(128, generator=g)
    W0, b0m, inv, gamma = u['self_posembed']
    sc = gamma * inv
    dW, db, dg, dbeta = fold.conv_bn_unfold(u['self_posembed'], dW1, db1)
    assert torch.equal(dW, dW1 * sc[:, None]) and torch.equal(db, db1 * sc)
    assert torch.equal(dg, ((dW1 * W0).sum(1) + db1 * b0m) * inv) and torch.equal(dbeta, db1)
