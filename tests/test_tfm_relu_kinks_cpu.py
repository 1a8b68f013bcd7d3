"""helpers.clear_relu_kinks on a reduced-depth Transformer (2 + 2 layers, d_model 64, d_ff 256): the shifted weights leave every ReLU
input of the step clear of the margin, move no bias by more than 1e-2 of its layer's RMS, touch nothing but the ReLU biases, and come out
the same on every run."""
import torch

from helpers import clear_relu_kinks, co, relu_inputs

V, D, DFF, LAYERS, F_ATT, HEADS = 60, 64, 256, 2, 96, 4
B, R, SPI, L = 4, 12, 5, 9
MARGIN = 8e-4


def _step():
    W = co.make_weights('transformer', V, D, DFF, LAYERS, 32, F_ATT, seed=3, logit_scale=3.0)
    _, att = co.make_inputs(B, R, 32, F_ATT, seed=5)
    g = torch.Generator().manual_seed(7)
    seq = torch.randint(1, V + 1, (B, SPI, L), generator=g)
    seq[..., 0] = 0
    for n in range(B * SPI):                                   # captions of 1 .. L - 1 words, then padding
        seq.view(-1, L)[n, 1 + n % (L - 1):] = 0
    regions = torch.ones(B, R)
    regions[1, 7:] = 0
    regions[3, 4:] = 0

    def forward(Wd):
        dt = Wd['att_embed.0.weight'].dtype
        return co.forward_teacher(co.Family('transformer', Wd, L, heads=HEADS), att.to(dt), att.to(dt), seq, regions)
    return W, att, forward


def _clearance(W, att, forward):
    """{layer: (smallest |input| / RMS, RMS)} of every ReLU of the step, in float64."""
    W64 = {k: v.double() for k, v in W.items()}
    return {n: (float(a.abs().min() / a.pow(2).mean().sqrt()), float(a.pow(2).mean().sqrt())) for n, a in relu_inputs(W64, att, forward)}


def test_clear_relu_kinks_reduced_depth():
    W, att, forward = _step()
    before = _clearance(W, att, forward)
    assert len(before) == 1 + 2 * LAYERS
    assert sum(c < MARGIN for c, _ in before.values()) >= 3               # the unshifted model has inputs inside the band
    out, shifted, largest = clear_relu_kinks(W, att, forward, MARGIN)
    print('units shifted per layer %s; largest shift %.2e x RMS' % (shifted, largest))
    assert sum(shifted.values()) > 0
    after = _clearance(out, att, forward)
    assert set(after) == set(before) == set(shifted)
    for name, (clear, _) in after.items():
        assert clear >= MARGIN, (name, clear)
    assert largest <= 1e-2
    bias_of = {'att_embed': 'att_embed.0.bias'}
    bias_of.update({'%s.layers.%d' % (s, i): 'model.%s.layers.%d.feed_forward.w_1.bias' % (s, i) for s in ('encoder', 'decoder') for i in range(LAYERS)})
    for name, key in bias_of.items():
        moved = (out[key].double() - W[key].double()).abs()
        assert float(moved.max()) <= 1e-2 * before[name][1], name
        assert int((moved > 0).sum()) == shifted[name], name
    for k in W:
        assert out[k].dtype == W[k].dtype
        if k not in bias_of.values():
            assert torch.equal(out[k], W[k]), k
    again = clear_relu_kinks(W, att, forward, MARGIN)
    assert again[1:] == (shifted, largest)
    assert all(torch.equal(again[0][k], out[k]) for k in out)
