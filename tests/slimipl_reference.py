"""Reference models of slimIPL's two kernels (recipes/slimIPL/src/Train.cpp:1663-1673, :1823-1831).

soft_label_loss: float64 over logits [..., N] (rows = every leading index),
    loss = -scale / rows * sum_rows sum_c p_c (z_c - lse(z)),   p = softmax(teacher),  z = student
    d_student = scale / rows * (softmax(z) - p)
ema_update: float32, rounded as w2l_ema_update rounds it: d and 1 - d each rounded once from double, then
    ema * d, params * (1 - d) and their sum each rounded once (NumPy float32 arithmetic, no fma)."""
import numpy as np


def _lse(x):
    m = x.max(axis=-1, keepdims=True)
    return m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True))


def soft_label_loss(student, teacher, scale):
    z = np.asarray(student, np.float64)
    t = np.asarray(teacher, np.float64)
    N = z.shape[-1]
    z, t = z.reshape(-1, N), t.reshape(-1, N)
    rows = z.shape[0]
    p = np.exp(t - _lse(t))
    logq = z - _lse(z)
    loss = -float(scale) / rows * float((p * logq).sum())
    d = float(scale) / rows * (np.exp(logq) - p)
    return loss, d.reshape(np.shape(student))


def ema_update(ema, params, decay):
    d, omd = np.float32(decay), np.float32(1.0 - float(decay))
    return np.asarray(ema, np.float32) * d + np.asarray(params, np.float32) * omd
