"""Outputs and device times of the memory-bound passes around the GEMMs: LayerNorm (two-pass, cooperative and per-row),
WeightNorm, GLU, axpy, column sums, the squared gradient norm and the SGD step.

Every pass has a float4 instance (V = 4) and a scalar one (V = 1); the float4 one runs when the lengths are multiples of 4
and the buffers are 16-byte aligned.  The cases below reach both: each entry point runs on aligned buffers and on buffers
that start one float into their allocation, at lengths that are and are not multiples of 4.

  python scripts/check_memory_passes.py --out outputs.npz [--root TREE]
      calls every entry point on seeded inputs and writes every output array to one .npz.  --root picks the source
      tree whose wav2letter_b200 package (and library) is imported, so two trees can be compared array by array.
  python scripts/check_memory_passes.py --compare a.npz b.npz
      exits 1 unless both files hold the same arrays, bit for bit (np.array_equal).
  python scripts/check_memory_passes.py --time [--root TREE]
      prints one JSON line per entry point: the median device ms of 20 calls (CUDA events), at the TDS training shapes
      (B = 16, 600 frames, 800 features) and conv_glu-sized WeightNorm / GLU rows.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np


def load(root):
    sys.path.insert(0, root)
    import torch
    from wav2letter_b200 import capi

    return torch, capi


def passes(torch, capi):
    """yields (name, thunk); a thunk runs one call and returns its output tensors"""
    lib, P, S = capi.lib, capi._ptr, capi._stream
    gen = torch.Generator(device="cuda").manual_seed(1234)

    def buf(n, off, fill=None):  # n floats starting `off` floats into a fresh allocation
        t = torch.randn(n + off, device="cuda", generator=gen) if fill is None else torch.full((n + off,), fill, device="cuda")
        return t[off:]

    def layernorm(B, R, off, res, affine):
        a = buf(B * R, off).clamp_min(0) * 1.3  # a ReLU branch output: has zeros for the masks
        r = buf(B * R, off) * 2 + 0.5 if res else None
        dy = buf(B * R, off)
        gain, bias = (torch.tensor([1.7], device="cuda"), torch.tensor([-0.3], device="cuda")) if affine else (None, None)
        y, mr = buf(B * R, off, 0.0), torch.empty(2 * B, device="cuda")
        scratch = capi.layernorm_scratch(B, "cuda")
        capi._check(lib.w2l_layernorm_fwd(S(), B, R, 1e-5, P(a), P(r), P(gain), P(bias), P(y), P(mr), P(scratch)))
        out = [y, mr]
        for mode in (0, 1, 2):
            d_branch, d_res = buf(B * R, off, 0.0), buf(B * R, off, 0.0) if res else None
            dg, db = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
            capi._check(lib.w2l_layernorm_bwd(S(), B, R, P(a), P(r), P(dy), P(gain), P(mr), P(d_branch), P(d_res), mode, 1.25,
                                              P(dg) if affine else None, P(db) if affine else None, P(scratch)))
            out += [d_branch] + ([d_res] if res else []) + ([dg, db] if affine else [])
        return out

    def layernorm_rows(G, R, off):
        a, r, y, mr = buf(G * R, off), buf(G * R, off), buf(G * R, off, 0.0), torch.empty(2 * G, device="cuda")
        gain, bias = torch.tensor([0.8], device="cuda"), torch.tensor([0.1], device="cuda")
        capi._check(lib.w2l_layernorm_rows_fwd(S(), G, R, 1e-5, P(a), P(r), P(gain), P(bias), P(y), P(mr)))
        return [y, mr]

    def weightnorm(rows, ln, off):
        v, g, dw = buf(rows * ln, off), torch.rand(rows, device="cuda", generator=gen) + 0.5, buf(rows * ln, off)
        w, inv = buf(rows * ln, off, 0.0), torch.empty(rows, device="cuda")
        dv, dg = buf(rows * ln, off), torch.randn(rows, device="cuda", generator=gen)  # the backward accumulates
        capi._check(lib.w2l_weightnorm_fwd(S(), rows, ln, P(v), P(g), P(w), P(inv)))
        capi._check(lib.w2l_weightnorm_bwd(S(), rows, ln, P(v), P(g), P(inv), P(dw), P(dv), P(dg)))
        return [w, inv, dv, dg]

    def glu(rows, H, p, off):
        x, dy, y, dx = buf(rows * 2 * H, off), buf(rows * H, off), buf(rows * H, off, 0.0), buf(rows * 2 * H, off, 0.0)
        capi._check(lib.w2l_glu_fwd(S(), rows, H, P(x), P(y), p, 77))
        capi._check(lib.w2l_glu_bwd(S(), rows, H, P(x), P(dy), P(dx), p, 77))
        return [y, dx]

    def axpy(n, off):
        x, y = buf(n, off), buf(n, off)
        capi._check(lib.w2l_axpy(S(), n, 0.37, P(x), P(y)))
        return [y]

    def colsum(M, N, ld, off):
        X, out = buf(M * ld, off), torch.ones(N, device="cuda")
        capi._check(lib.w2l_colsum_accumulate(S(), M, N, P(X), ld, P(out)))
        return [out]

    def norm_sgd(n, nesterov):
        p, g, v = buf(n, 0), buf(n, 0), buf(n, 0)
        sq = torch.full((1,), 0.5, dtype=torch.float64, device="cuda")
        capi._check(lib.w2l_sq_norm_accumulate(S(), n, P(g), P(sq)))
        capi._check(lib.w2l_sgd_step_ex(S(), n, P(p), P(g), P(v), 0.1, 0.9, 1e-3, 0.25, 1.0, P(sq), nesterov, None))
        return [sq, p, v]

    # the shapes of tests/test_gpu_am_kernels.py::test_layernorm_fwd_bwd: two-pass, cooperative and per-row paths
    for B, R in [(1, 17), (3, 5000), (4, 50 * 800), (2, 250 * 1440), (2400, 1200), (1500, 2160), (1300, 30)]:
        for off in (0, 1):
            for res, affine in ((True, True), (True, False), (False, True), (False, False)):
                yield f"layernorm_B{B}_R{R}_off{off}_res{int(res)}_aff{int(affine)}", lambda B=B, R=R, o=off, re=res, af=affine: layernorm(B, R, o, re, af)
    for G, R, off in [(1000, 800, 0), (1000, 800, 1), (333, 30, 0), (333, 77, 0)]:
        yield f"layernorm_rows_G{G}_R{R}_off{off}", lambda G=G, R=R, o=off: layernorm_rows(G, R, o)
    for ln in (528, 530):
        for off in (0, 1):
            yield f"weightnorm_len{ln}_off{off}", lambda ln=ln, o=off: weightnorm(37, ln, o)
    for H in (120, 122):
        for p in (0.0, 0.3):
            for off in (0, 1):
                yield f"glu_H{H}_p{p}_off{off}", lambda H=H, p=p, o=off: glu(501, H, p, o)
    for n in (100000, 100003):
        for off in (0, 1):
            yield f"axpy_n{n}_off{off}", lambda n=n, o=off: axpy(n, o)
    for M, N, ld, off in [(1000, 77, 77, 0), (2403, 1000, 1120, 0), (2403, 1000, 1120, 1), (9600, 800, 800, 0)]:
        yield f"colsum_M{M}_N{N}_ld{ld}_off{off}", lambda M=M, N=N, ld=ld, o=off: colsum(M, N, ld, o)
    for n in (100003, 1 << 20):
        for nesterov in (0, 1):
            yield f"sqnorm_sgd_n{n}_nesterov{nesterov}", lambda n=n, ne=nesterov: norm_sgd(n, ne)


def timed(torch, capi):
    """(name, thunk) at the benchmarked shapes; a thunk makes one call"""
    lib, P, S = capi.lib, capi._ptr, capi._stream
    B, R = 16, 600 * 800
    a, r, dy, y, d_b, d_r = (torch.randn(B * R, device="cuda") for _ in range(6))
    G, F = 16 * 600, 800  # the same activations as per-frame groups (per-row LayerNorm)
    mr, gain, bias = torch.empty(2 * G, device="cuda"), torch.ones(1, device="cuda"), torch.zeros(1, device="cuda")
    dg, db, scratch = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda"), capi.layernorm_scratch(G, "cuda")
    rows, ln = 1000, 12000
    v, w, dv = (torch.randn(rows * ln, device="cuda") for _ in range(3))
    g, inv, dgn = torch.rand(rows, device="cuda") + 0.5, torch.empty(rows, device="cuda"), torch.zeros(rows, device="cuda")
    gr, H = 8 * 1000, 1000
    x, gy, gdy, gdx = torch.randn(gr * 2 * H, device="cuda"), torch.empty(gr * H, device="cuda"), torch.randn(gr * H, device="cuda"), torch.empty(gr * 2 * H, device="cuda")
    n = 16 << 20
    p, pg, pv, sq = torch.randn(n, device="cuda"), torch.randn(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(1, dtype=torch.float64, device="cuda")
    colsum_out = torch.zeros(F, device="cuda")
    yield "layernorm_fwd", lambda: lib.w2l_layernorm_fwd(S(), B, R, 1e-5, P(a), P(r), P(gain), P(bias), P(y), P(mr), P(scratch))
    yield "layernorm_bwd", lambda: lib.w2l_layernorm_bwd(S(), B, R, P(a), P(r), P(dy), P(gain), P(mr), P(d_b), P(d_r), 1, 1.25, P(dg), P(db), P(scratch))
    yield "layernorm_rows_fwd", lambda: lib.w2l_layernorm_rows_fwd(S(), G, F, 1e-5, P(a), P(r), P(gain), P(bias), P(y), P(mr))
    yield "layernorm_rows_bwd", lambda: lib.w2l_layernorm_bwd(S(), G, F, P(a), P(r), P(dy), P(gain), P(mr), P(d_b), P(d_r), 1, 1.25, P(dg), P(db), P(scratch))
    yield "weightnorm_fwd", lambda: lib.w2l_weightnorm_fwd(S(), rows, ln, P(v), P(g), P(w), P(inv))
    yield "weightnorm_bwd", lambda: lib.w2l_weightnorm_bwd(S(), rows, ln, P(v), P(g), P(inv), P(w), P(dv), P(dgn))
    yield "glu_fwd", lambda: lib.w2l_glu_fwd(S(), gr, H, P(x), P(gy), 0.2, 5)
    yield "glu_bwd", lambda: lib.w2l_glu_bwd(S(), gr, H, P(x), P(gdy), P(gdx), 0.2, 5)
    yield "axpy", lambda: lib.w2l_axpy(S(), n, 0.5, P(pg), P(pv))
    yield "colsum_accumulate", lambda: lib.w2l_colsum_accumulate(S(), G, F, P(a), F, P(colsum_out))
    yield "sq_norm_accumulate", lambda: lib.w2l_sq_norm_accumulate(S(), n, P(pg), P(sq))
    yield "sgd_step_ex", lambda: lib.w2l_sgd_step_ex(S(), n, P(p), P(pg), P(pv), 1e-6, 0.9, 0.0, 1.0, 1.0, P(sq), 0, None)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    ap.add_argument("--time", action="store_true")
    args = ap.parse_args()
    if args.compare:
        a, b = (np.load(f) for f in args.compare)
        bad = sorted(set(a.files) ^ set(b.files)) + [k for k in a.files if k in b.files and not np.array_equal(a[k], b[k])]
        cases = sorted({k.split(":")[0] for k in bad})
        print(f"{len(a.files)} arrays compared, {len(bad)} differ" + (" in: " + " ".join(cases) if bad else ""))
        sys.exit(1 if bad else 0)
    torch, capi = load(args.root)
    if args.time:
        for name, call in timed(torch, capi):
            for _ in range(3):
                capi._check(call())
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(40)]
            for i in range(20):
                ev[2 * i].record()
                capi._check(call())
                ev[2 * i + 1].record()
            torch.cuda.synchronize()
            ms = sorted(ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(20))
            print(json.dumps({"pass": name, "median_ms": round(ms[10], 4), "min_ms": round(ms[0], 4)}))
        return
    arrays = {}
    for name, run in passes(torch, capi):
        for k, t in enumerate(run()):
            arrays[f"{name}:{k}"] = t.cpu().numpy()
    np.savez(args.out, **arrays)
    print(f"{len(arrays)} arrays -> {args.out}")


if __name__ == "__main__":
    main()
