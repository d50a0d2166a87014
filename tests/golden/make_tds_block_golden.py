"""Extracts the known-answer vectors of the reference's own TDS-block test
(recipes/streaming_convnets/inference/inference/module/test/TDSBlockTest.cpp:27-188, TEST(TDSBlock, TestOne):
T=10, groups=5, 2 channels per group, kernel 3, padding 1/1, tolerance 1e-2) into tests/golden/tds_block_golden.npz.
Run once with the root of the reference tree as its argument; only the numbers are stored (test data).

Layout of the reference's inference modules (Conv1dTest.cpp:30-104, TDSBlockTest.cpp): activations [T][groups][c]
(feature index w*C + c), conv weights [cout/g][kw][cin/g] shared by every group, Linear weights W[i*nOut + o],
LayerNorm per frame over all features with scalar affine.  Before writing, the script re-derives the expected output
with numpy (block = LN(x + ReLU(conv(x))) -> LN(h + lin2(ReLU(lin1(h))))) and refuses to write unless it agrees with
the reference's numbers within the reference's own tolerance."""
import os
import re
import sys

import numpy as np

SRC = "recipes/streaming_convnets/inference/inference/module/test/TDSBlockTest.cpp"  # inside the reference tree


def main(ref_root):
    text = open(os.path.join(ref_root, SRC)).read()
    body = text[text.index("TEST(TDSBlock, TestOne)"):text.index("TEST(TDSBlock, Serialization)")]
    vec = {}
    for m in re.finditer(r"std::vector<float>\s+(\w+)\s*=\s*\{([^}]*)\}", body):
        vec[m.group(1)] = np.array([float(v) for v in m.group(2).replace("\n", " ").split(",") if v.strip()], dtype=np.float32)
    T, W, C, K = 10, 5, 2, 3
    x = vec["in"].reshape(T, W, C)
    cw = vec["conv_weights"].reshape(C, K, C)  # [cout][kw][cin]
    cb = vec["conv_bias"]
    nf = W * C

    def ln(v):
        m = v.mean(axis=-1, keepdims=True)
        s = np.sqrt(np.maximum((v * v).mean(axis=-1, keepdims=True) - m * m, 0))
        return (v - m) / s

    xp = np.pad(x.astype(np.float64), ((1, 1), (0, 0), (0, 0)))
    conv = np.zeros((T, W, C))
    for t in range(T):
        for dk in range(K):
            conv[t] += xp[t + dk] @ cw[:, dk, :].T.astype(np.float64)
    conv += cb
    h = ln((x + np.maximum(conv, 0)).reshape(T, nf))
    W1 = vec["lin1_weights"].reshape(nf, nf).astype(np.float64)  # W[i*nOut + o]
    W2 = vec["lin2_weights"].reshape(nf, nf).astype(np.float64)
    u = np.maximum(h @ W1 + vec["lin1_bias"], 0) @ W2 + vec["lin2_bias"]
    out = ln(h + u)
    exp = vec["expectedOutput"].reshape(T, nf)
    err = float(np.abs(out - exp).max())
    print("numpy re-derivation vs the reference's expectedOutput: max abs error", err)
    if err > 1e-2:
        sys.exit("layout assumption does not reproduce the reference's golden")
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tds_block_golden.npz")
    np.savez_compressed(path, T=T, W=W, C=C, K=K, pad_left=1, pad_right=1, **{k: v for k, v in vec.items() if k != "inputValues"})
    print("wrote", path)


if __name__ == "__main__":
    main(sys.argv[1])
