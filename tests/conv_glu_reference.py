"""Plain torch model of the conv_glu large-channel convolution's operand contracts (include/w2l_b200.h, "Conv1D + GLU
family"), for tests/test_gpu_conv_glu_layers.py and tests/test_conv_glu_reference_cpu.py.

  pad_row(kind, n)        the padded row length fl::Conv2D::forwardGemm uses: a multiple of 4 floats in f32 / tf32 mode,
                          of 8 elements in bf16 / fp16 mode
  padded_sizes(...)       (Cp, CoutP) as forwardGemm computes them: Cp = pad_row(cin), CoutP = 2 pad_row(cout / 2) with a
                          GLU (each half padded on its own), pad_row(cout) without
  out_rows(...)           row of the padded operand that holds each output channel
  arrange(...)            w [cout][cin][kw], bias -> fwd [cout_p][kw*cin_p] (k = dk*cin_p + ci), flip [cin_p][kw*cout_p]
                          (k = j*cout_p + row(co), tap kw-1-j) and bias_p [cout_p]; every padded entry is 0
  unarrange(...)          the reverse gather: dw[co][ci][dk] = dfwd[row(co)][dk*cin_p + ci]
  conv_glu_layers(nfeat)  every (cin, cout, kw, pad) of archs.conv_glu_wsj() and archs.conv_glu_librispeech()

Every function only moves values, so it works on any dtype and device and is exact.
"""
from __future__ import annotations

import importlib.util
import os
import re

import torch
import torch.nn.functional as F
from torch.nn.grad import conv1d_weight

# archs.py by path: pure Python, so the CPU tests never map the CUDA library
_spec = importlib.util.spec_from_file_location("w2l_archs", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                                         "wav2letter_b200", "archs.py"))
archs = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(archs)

KINDS = ("f32", "tf32", "bf16", "fp16")


def pad_row(kind: str, n: int) -> int:
    q = 8 if kind in ("bf16", "fp16") else 4
    return (n + q - 1) // q * q


def padded_sizes(kind: str, cin: int, cout: int, glu_split: bool) -> tuple[int, int]:
    return pad_row(kind, cin), (2 * pad_row(kind, cout // 2) if glu_split else pad_row(kind, cout))


def out_rows(cout: int, cout_p: int, glu_split: bool, device=None) -> torch.Tensor:
    co = torch.arange(cout, device=device)
    if not glu_split:
        return co
    h, hp = cout // 2, cout_p // 2
    return torch.where(co < h, co, hp + (co - h))


def arrange(w: torch.Tensor, bias: torch.Tensor | None, cin_p: int, cout_p: int, glu_split: bool):
    cout, cin, kw = w.shape
    rows = out_rows(cout, cout_p, glu_split, w.device)
    fwd = torch.zeros(cout_p, kw, cin_p, dtype=w.dtype, device=w.device)
    fwd[rows, :, :cin] = w.permute(0, 2, 1)  # fwd[row(co)][dk][ci] = w[co][ci][dk]
    flip = torch.zeros(cin_p, kw, cout_p, dtype=w.dtype, device=w.device)
    flip[:cin, :, rows] = w.flip(2).permute(1, 2, 0)  # flip[ci][j][row(co)] = w[co][ci][kw-1-j]
    bias_p = None
    if bias is not None:
        bias_p = torch.zeros(cout_p, dtype=bias.dtype, device=bias.device)
        bias_p[rows] = bias
    return fwd.reshape(cout_p, kw * cin_p), flip.reshape(cin_p, kw * cout_p), bias_p


def unarrange(dfwd: torch.Tensor, cin: int, cout: int, kw: int, cin_p: int, cout_p: int, glu_split: bool) -> torch.Tensor:
    rows = out_rows(cout, cout_p, glu_split, dfwd.device)
    return dfwd.view(cout_p, kw, cin_p)[rows, :, :cin].permute(0, 2, 1).contiguous()


def conv_glu_layers(nfeat: int) -> list[tuple[int, int, int, int]]:
    """(cin, cout, kw, pad) of every `WN 3 C cin cout kw 1 pad` layer of both conv_glu recipes (pad -1: SAME)"""
    out = []
    for gen in (archs.conv_glu_wsj, archs.conv_glu_librispeech):
        for m in re.finditer(r"^WN 3 C (\S+) (\d+) (\d+) 1 (-?\d+)$", gen(), re.M):
            cin = nfeat if m.group(1) == "NFEAT" else int(m.group(1))
            out.append((cin, int(m.group(2)), int(m.group(3)), int(m.group(4))))
    return out


def im2col(x: torch.Tensor, kw: int) -> torch.Tensor:
    """x [T][C] -> [T-kw+1][kw*C]: row t is frames t .. t+kw-1 back to back (the GEMM's overlapping-row view)"""
    T, C = x.shape
    return x.as_strided((T - kw + 1, kw * C), (C, 1))


# ---------------------------------------------------------------------------------------------------------------------------
# The trainer's conv_glu network in float64, with a first-order bound on the error of the GPU result of every tensor.
#
# Each GEMM of the trainer (conv forward, weight gradient, data gradient; the Linear head's three) rounds its operands to
# the precision mode's operand type and accumulates in fp32, so |C - ref| <= c (|A| |B|) element-wise, with
#   f32  (3xTF32)   c = 4e-6     the element-wise bound of test_gpu_gemm.py's f32x3 test
#   tf32 / fp16     c = 1.5e-3   11 significant bits per operand: 2 * 2^-11 per product, plus fp32 accumulation
#   bf16            c = 6e-3     8 significant bits: the same derivation with 2 * 2^-9
# fp16 operands also round below 2^-14 onto the subnormal grid, an absolute error of at most 2^-25 per operand element.
# Errors already in an operand pass through the contraction with the other operand's magnitudes, so every tensor T
# carries E_T and every product adds c (|A| |B|) + E_A |B| + |A| E_B.  Around the GEMMs: WeightNorm's fp32 norm
# (a block sum of len terms: (len / 1024 + 16) ulps), GLU's __expf sigmoid ((6 + 1.2 |s|) ulps, twice that in the backward,
# where sigma' = sg (1 - sg) also keeps sg's absolute rounding when the gate saturates; the sigmoid's response to an error
# in s is bounded over the whole interval s +- E_s, not linearised),
# the bias add in the GEMM epilogue (1 ulp) and the bias gradients' fp32 sums over `rows` terms (rows ulps of sum |dy|).
# ---------------------------------------------------------------------------------------------------------------------------
#
# Largest measured |err| / (1.25 x bound) on an H100 80GB HBM3 at its 700 W limit, over the trainer cases of
# test_gpu_conv_glu_layers.py (emissions; conv v, g, bias; head v, g, bias):
#   f32   0.12;  0.66, 0.011, 0.57;  0.43, 0.044, 0.21
#   tf32  0.02;  0.39, 0.031, 0.14;  0.091, 0.009, 0.26
#   bf16  0.05;  0.66, 0.063, 0.22;  0.12, 0.0031, 0.32
#   fp16  0.027; 0.37, 0.031, 0.12;  0.073, 0.0089, 0.34
# The f32 weight-gradient GEMM alone at these shapes (K = B Ts rows up to 1908) measures 0.51 of c |A| |B|: c needs no K term.
U32 = 2.0 ** -24
GEMM_C = {"f32": 4e-6, "tf32": 1.5e-3, "fp16": 1.5e-3, "bf16": 6e-3}
FP16_FLOOR = 2.0 ** -25


def _wn(v, g):
    n = v.flatten(1).norm(dim=1)
    shape = (-1,) + (1,) * (v.dim() - 1)
    w = (g / n).view(shape) * v
    cwn = (v[0].numel() / 1024 + 16) * U32
    return w, cwn * w.abs(), n, cwn


def _wn_bwd(v, g, n, cwn, dw, Edw):
    shape = (-1,) + (1,) * (v.dim() - 1)
    dot = (dw * v).flatten(1).sum(1)
    adot = (dw.abs() * v.abs()).flatten(1).sum(1)
    Edot = (Edw * v.abs()).flatten(1).sum(1) + cwn * adot
    dg = dot / n
    dv = (g / n).view(shape) * (dw - v * (dot / n ** 2).view(shape))
    Edg = Edot / n
    Edv = (g.abs() / n).view(shape) * (Edw + v.abs() * (Edot / n ** 2).view(shape) + cwn * (dw.abs() + v.abs() * (adot / n ** 2).view(shape)))
    return dv, Edv, dg, Edg


class ConvGluNet:
    """`WN 3 C cin cout kw 1 pad` + `GLU 2` per layer, `RO 2 0 3 1`, `WN 0 L C N`: parameters [v, g, b] per layer and for
    the head (the trainer's flat-arena order), float64.  forward(x [B, cin, T]) -> z [B, T', N]; backward(G) -> [(grad,
    bound)] per parameter.  Every value comes with its bound for the precision mode `kind`."""

    def __init__(self, params, layers, kind):
        self.p, self.layers, self.c = params, layers, GEMM_C[kind]
        self.floor = FP16_FLOOR if kind == "fp16" else 0.0

    def _lin(self, f, a, Ea, b, Eb, *args):
        """f bilinear: value f(a, b) and its bound c f(|a|, |b|) + f(Ea, |b|) + f(|a|, Eb) (+ the fp16 grid floor)"""
        val = f(a, b, *args)
        E = self.c * f(a.abs(), b.abs(), *args) + f(Ea, b.abs(), *args) + f(a.abs(), Eb, *args)
        if self.floor:
            E = E + self.floor * (f(torch.ones_like(a), b.abs(), *args) + f(a.abs(), torch.ones_like(b), *args))
        return val, E

    def forward(self, x):
        self.saved = []
        Ex = torch.zeros_like(x)
        for i, (cin, cout, kw, pad) in enumerate(self.layers):
            v, g, b = (t.view(cout, cin, kw) if j == 0 else t for j, t in enumerate(self.p[3 * i:3 * i + 3]))
            w, Ew, n, cwn = _wn(v, g)
            pl = kw // 2 if pad < 0 else pad
            xp, Exp = F.pad(x, (pl, pl)), F.pad(Ex, (pl, pl))
            y, Ey = self._lin(F.conv1d, xp, Exp, w, Ew)
            y = y + b.view(-1, 1)
            Ey = Ey + self.c * b.abs().view(-1, 1) + U32 * y.abs()
            H = cout // 2
            a, s, Ea, Es = y[:, :H], y[:, H:], Ey[:, :H], Ey[:, H:]
            sg = torch.sigmoid(s)
            ds = sg * (1 - sg)
            # not linearised: where the sigmoid saturates, 16-bit operands can move s by more than 1.  sigma' is largest
            # nearest 0 and bounds |sigma''|, so over [s - Es, s + Es] both sigma and sigma' move by at most dmax Es
            sm = torch.sigmoid((s.abs() - Es).clamp(min=0))
            Esg = sm * (1 - sm) * Es
            x = a * sg
            Ex = sg * Ea + (a.abs() + Ea) * Esg + (6 + 1.2 * s.abs()) * U32 * x.abs()
            self.saved.append((v, g, w, Ew, n, cwn, xp, Exp, a, s, Ea, Esg, sg, ds, pl))
        h, Eh = x.permute(0, 2, 1), Ex.permute(0, 2, 1)  # RO 2 0 3 1: [B, T', C]
        v2, g2, b2 = self.p[-3:]
        N = g2.numel()
        v2 = v2.view(N, -1)
        w2, Ew2, n2, cwn2 = _wn(v2, g2)
        z, Ez = self._lin(lambda p, q: p @ q.t(), h, Eh, w2, Ew2)
        z = z + b2
        Ez = Ez + self.c * b2.abs() + U32 * z.abs()
        self.head = (v2, g2, w2, Ew2, n2, cwn2, h, Eh)
        return z, Ez

    def backward(self, G, EG=None):
        EG = torch.zeros_like(G) if EG is None else EG
        self.dweights = []  # per conv layer: the weight gradient, its bound, dy and the padded input
        v2, g2, w2, Ew2, n2, cwn2, h, Eh = self.head
        dw2, Edw2 = self._lin(lambda p, q: torch.einsum("btn,btc->nc", p, q), G, EG, h, Eh)
        db2 = G.sum((0, 1))
        Edb2 = G[..., 0].numel() * U32 * G.abs().sum((0, 1)) + EG.sum((0, 1))
        dh, Edh = self._lin(lambda p, q: p @ q, G, EG, w2, Ew2)
        dv2, Edv2, dg2, Edg2 = _wn_bwd(v2, g2, n2, cwn2, dw2, Edw2)
        out = [(db2, Edb2), (dg2, Edg2), (dv2, Edv2)]  # reversed below
        dx, Edx = dh.permute(0, 2, 1), Edh.permute(0, 2, 1)
        for (cin, cout, kw, pad), (v, g, w, Ew, n, cwn, xp, Exp, a, s, Ea, Esg, sg, ds, pl) in zip(reversed(self.layers), reversed(self.saved)):
            dA = dx * sg
            EdA = Edx * (sg + Esg) + dx.abs() * Esg + (6 + 1.2 * s.abs()) * U32 * dA.abs()
            dS = dx * a * ds
            # the kernel forms sigma' as sg * (1 - sg): where the gate saturates, 1 - sg cancels and keeps sg's absolute
            # rounding, (6 + 1.2 |s|) ulps of sg, however small sigma' is
            EdS = (Edx * (a.abs() + Ea) * (ds + Esg) + dx.abs() * (ds * Ea + (a.abs() + Ea) * Esg)
                   + (12 + 2.4 * s.abs()) * U32 * dS.abs() + dx.abs() * (a.abs() + Ea) * sg * (6 + 1.2 * s.abs()) * U32)
            dy, Edy = torch.cat([dA, dS], 1), torch.cat([EdA, EdS], 1)
            dw, Edw = self._lin(lambda p, q: conv1d_weight(p, w.shape, q), xp, Exp, dy, Edy)
            rows = dy.shape[0] * xp.shape[2]  # the bias gradient sums every row of the batch, slack rows included
            db = dy.sum((0, 2))
            Edb = rows * U32 * dy.abs().sum((0, 2)) + Edy.sum((0, 2))
            dxp, Edxp = self._lin(lambda p, q: F.conv_transpose1d(p, q), dy, Edy, w, Ew)
            T = xp.shape[2] - 2 * pl
            dx, Edx = dxp[..., pl:pl + T], Edxp[..., pl:pl + T]
            self.dweights.insert(0, (dw, Edw, dy, xp))
            dv, Edv, dg, Edg = _wn_bwd(v, g, n, cwn, dw, Edw)
            out += [(db, Edb), (dg, Edg), (dv.flatten(), Edv.flatten())]
        return [(t.flatten(), e.flatten()) for t, e in reversed(out)]
