"""The operand model of tests/conv_glu_reference.py is the convolution: the im2col rows of an input times the arranged
forward operand are torch's conv1d, and the flipped operand on dY with kw-1 zero frames in front is conv1d's input
gradient (float64, CPU)."""
import pytest
import torch
import torch.nn.functional as F

from conv_glu_reference import arrange, conv_glu_layers, im2col, out_rows, pad_row, padded_sizes, unarrange


@pytest.mark.parametrize("cin,cout,kw,glu,kind", [(5, 6, 3, False, "f32"), (7, 10, 4, True, "f32"), (9, 26, 5, True, "bf16"),
                                                   (1, 2, 1, True, "fp16"), (33, 14, 2, True, "tf32"), (12, 9, 6, False, "bf16")])
def test_arranged_operands_are_the_convolution(cin, cout, kw, glu, kind):
    g = torch.Generator().manual_seed(cin * 100 + cout)
    cin_p, cout_p = padded_sizes(kind, cin, cout, glu)
    assert cin_p % 4 == 0 and cout_p % 4 == 0 and cin_p >= cin and cout_p >= cout
    if glu:
        assert cout_p % 8 == 0 and cout_p // 2 >= cout // 2
    T = 3 * kw + 7
    w = torch.randn(cout, cin, kw, dtype=torch.float64, generator=g)
    b = torch.randn(cout, dtype=torch.float64, generator=g)
    fwd, flip, bias_p = arrange(w, b, cin_p, cout_p, glu)
    rows = out_rows(cout, cout_p, glu)
    pad = torch.ones(cout_p, dtype=torch.bool)
    pad[rows] = False
    assert not fwd[pad].count_nonzero() and not bias_p[pad].count_nonzero() and not flip.view(cin_p, kw, cout_p)[..., pad].count_nonzero()
    assert not fwd.view(cout_p, kw, cin_p)[..., cin:].count_nonzero() and not flip[cin:].count_nonzero()

    x = torch.zeros(T, cin_p, dtype=torch.float64)
    x[:, :cin] = torch.randn(T, cin, dtype=torch.float64, generator=g)
    y = im2col(x, kw) @ fwd.t() + bias_p  # [Tout][cout_p]
    xr = x[:, :cin].t().unsqueeze(0).requires_grad_(True)
    ref = F.conv1d(xr, w, b)[0].t()  # [Tout][cout]
    torch.testing.assert_close(y[:, rows], ref, rtol=1e-12, atol=1e-12)
    assert not y[:, pad].count_nonzero()

    dy = torch.randn(T - kw + 1, cout, dtype=torch.float64, generator=g)
    ref.backward(dy)
    dyp = torch.zeros(T + kw - 1, cout_p, dtype=torch.float64)  # kw-1 zero frames either side
    dyp[kw - 1:T, rows] = dy
    dx = im2col(dyp, kw) @ flip.t()  # [T][cin_p]
    torch.testing.assert_close(dx[:, :cin], xr.grad[0].t(), rtol=1e-12, atol=1e-12)
    assert not dx[:, cin:].count_nonzero()

    # the weight gradient of the arranged operand, gathered back, is conv1d's weight gradient
    w_ = w.clone().requires_grad_(True)
    F.conv1d(x[:, :cin].t().unsqueeze(0), w_).backward(dy.t().unsqueeze(0))
    dyf = torch.zeros(T - kw + 1, cout_p, dtype=torch.float64)
    dyf[:, rows] = dy
    dfwd = dyf.t() @ im2col(x, kw)  # [cout_p][kw*cin_p]
    torch.testing.assert_close(unarrange(dfwd, cin, cout, kw, cin_p, cout_p, glu), w_.grad, rtol=1e-12, atol=1e-12)


def test_padded_sizes_follow_the_precision_modes():
    assert [pad_row(k, 321) for k in ("f32", "tf32", "bf16", "fp16")] == [324, 324, 328, 328]
    # odd GLU halves: each half is padded on its own, so the second half starts past the first's padding
    assert padded_sizes("f32", 621, 1366, True) == (624, 1368) and padded_sizes("bf16", 621, 1366, True) == (624, 1376)
    assert padded_sizes("f32", 40, 1366, False)[1] == 1368
    assert out_rows(1366, 1368, True)[683].item() == 684


def test_layer_list_is_both_recipes():
    assert len(conv_glu_layers(40)) == 15 + 17
    assert conv_glu_layers(80)[15] == (80, 400, 13, 170) and conv_glu_layers(40)[0] == (40, 200, 13, -1)
    assert conv_glu_layers(40)[-1] == (826, 1816, 29, 0)


@pytest.mark.parametrize("kind", ["f32", "fp16"])
def test_bounded_network_values_are_autograds(kind):
    """ConvGluNet's hand-written forward and backward are torch autograd's, and its bounds are finite and non-negative"""
    from conv_glu_reference import ConvGluNet

    g = torch.Generator().manual_seed(7)
    layers = [(6, 10, 3, 2), (5, 8, 4, 0)]
    N, B, T = 4, 2, 9
    shapes = []
    for cin, cout, kw, _ in layers:
        shapes += [(cout * cin * kw,), (cout,), (cout,)]
    shapes += [(N * 4,), (N,), (N,)]
    params = [torch.randn(s, dtype=torch.float64, generator=g) for s in shapes]
    x = torch.randn(B, 6, T, dtype=torch.float64, generator=g)
    net = ConvGluNet(params, layers, kind)
    z, Ez = net.forward(x)
    G = torch.randn(z.shape, dtype=torch.float64, generator=g)
    grads = net.backward(G)

    p = [t.clone().requires_grad_(True) for t in params]
    h = x
    for i, (cin, cout, kw, pad) in enumerate(layers):
        v, gg, b = p[3 * i].view(cout, cin, kw), p[3 * i + 1], p[3 * i + 2]
        w = gg.view(-1, 1, 1) * v / v.reshape(cout, -1).norm(dim=1).view(-1, 1, 1)
        h = F.glu(F.conv1d(F.pad(h, (pad, pad)), w, b), dim=1)
    v, gg, b = p[-3].view(N, -1), p[-2], p[-1]
    zr = h.permute(0, 2, 1) @ (gg.view(-1, 1) * v / v.norm(dim=1, keepdim=True)).t() + b
    zr.backward(G)
    torch.testing.assert_close(z, zr, rtol=1e-12, atol=1e-12)
    assert bool((Ez > 0).all())
    for (d, E), t in zip(grads, p):
        torch.testing.assert_close(d, t.grad, rtol=1e-10, atol=1e-12)
        assert bool((E >= 0).all()) and bool(E.isfinite().all())
