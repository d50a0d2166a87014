"""float64 torch reference for archs of convolutions over features-as-channels with PReLU (the TIMIT recipe's
`V -1 1 NFEAT 0`, `C2 cin cout kw 1 1 1 -1 0`, `PR`, `DO 0`, `RO 2 0 3 1`, `L`): the opcodes the arch parity tests of
tests/test_gpu_prelu.py and tests/test_gpu_learnable_frontend.py run.  Parameters come from the trainer's flat arena in
module order: C2 w memory [cout][cin][kw], b [cout]; PR a [1]; L W memory [nOut][nIn], b [nOut].

PReLU (fl::PReLU, flashlight 0.3, recalled): y = x >= 0 ? x : a x; dy/da = x where x < 0."""
import torch
import torch.nn.functional as F


def prelu(x, a):
    return torch.where(x >= 0, x, a * x)


class ChannelNet:
    def __init__(self, arch_text, n_feat, n_label, flat, layout, dtype=torch.float64):
        self.ops = [ln.split("#")[0].replace("NFEAT", str(n_feat)).replace("NLABEL", str(n_label)).split()
                    for ln in arch_text.splitlines()]
        self.ops = [p for p in self.ops if p]
        self.params = [flat[o:o + n].detach().to(dtype).clone().requires_grad_(True) for o, n, _ in layout]
        self.dtype = dtype

    def forward(self, feat):
        """feat [B,1,F,T] -> emissions [B,T,N]"""
        it = iter(self.params)
        x = None
        for p in self.ops:
            op = p[0]
            if op == "V":
                assert x is None and p[2] == "1", "only the features-as-channels head view"
                x = feat.to(self.dtype)[:, 0].permute(0, 2, 1)  # [B,T,F]
            elif op == "C2":
                cin, cout, k = int(p[1]), int(p[2]), int(p[3])
                assert int(p[5]) == 1 and int(p[7]) == -1, "stride 1, SAME padding"
                w, b = next(it).view(cout, cin, k), next(it)
                x = F.conv1d(F.pad(x.permute(0, 2, 1), (k // 2, k // 2)), w, b).permute(0, 2, 1)
            elif op == "PR":
                x = prelu(x, next(it))
            elif op == "DO":
                assert float(p[1]) == 0.0, "dropout must be 0"
            elif op == "RO":
                pass
            elif op == "L":
                nin, nout = int(p[1]), int(p[2])
                W, b = next(it).view(nout, nin), next(it)
                x = F.linear(x, W, b)
            else:
                raise ValueError(f"opcode {op} not covered")
        assert next(it, None) is None, "arch / layout mismatch"
        return x

    def grads_flat(self, layout, total):
        out = torch.zeros(total, dtype=self.dtype, device=self.params[0].device)
        for (o, n, _), q in zip(layout, self.params):
            if q.grad is not None:
                out[o:o + n] = q.grad.reshape(-1)
        return out
