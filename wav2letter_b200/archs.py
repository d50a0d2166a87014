"""Architecture files of the four BASELINE.json model configs, generated from their layer tables.

Pure Python, no imports: bench.py's reference arm loads this file by path so that the CUDA library is never mapped
into the reference process.  tests/test_archs.py checks that every generator reproduces the recipe's arch file
token for token (stored in tests/golden/reference_archs.json):

  conv_glu_wsj()          recipes/conv_glu/wsj/network.arch              (configs[0])
  seq2seq_tds(ctc_head)   recipes/seq2seq_tds/librispeech/network.arch   (configs[1]; ctc_head swaps the encoder's
                                                                           `L 1440 1024` for `L 1440 NLABEL`)
  conv_glu_librispeech()  recipes/conv_glu/librispeech/network.arch      (configs[2])
  streaming_tds()         recipes/streaming_convnets/librispeech/am_500ms_future_context.arch   (configs[3])

and, outside the BASELINE configs (so outside BASELINE_ARCHS / REFERENCE_FILES, which bench.py and test_archs.py walk):

  learnable_frontend_timit()  recipes/learnable_frontend/am_baseline_conv_relu.arch  (TIMIT phones; checked against
                              tests/golden/learnable_frontend_arch.json)
"""


def _num(x):
    return repr(x) if isinstance(x, float) else str(x)


def conv_glu_wsj():
    layers = [("NFEAT", 200, 13), (100, 200, 3), (100, 200, 4), (100, 250, 5), (125, 250, 6), (125, 300, 7), (150, 350, 8),
              (175, 400, 9), (200, 450, 10), (225, 500, 11), (250, 500, 12), (250, 500, 13), (250, 600, 14), (300, 600, 15),
              (300, 750, 21)]
    out = ["V -1 1 NFEAT 0"]
    for cin, cout, kw in layers:
        out += [f"WN 3 C {cin} {cout} {kw} 1 -1", "GLU 2", "DO 0.25"]
    out += ["RO 2 0 3 1", "WN 0 L 375 1000", "GLU 0", "DO 0.25", "WN 0 L 500 NLABEL"]
    return "\n".join(out) + "\n"


def conv_glu_librispeech():
    layers = [("NFEAT", 400, 13, "0.2"), (200, 440, 14, "0.214"), (220, 484, 15, "0.22898"), (242, 532, 16, "0.2450086"),
              (266, 584, 17, "0.262159202"), (292, 642, 18, "0.28051034614"), (321, 706, 19, "0.30014607037"),
              (353, 776, 20, "0.321156295296"), (388, 852, 21, "0.343637235966"), (426, 936, 22, "0.367691842484"),
              (468, 1028, 23, "0.393430271458"), (514, 1130, 24, "0.42097039046"), (565, 1242, 25, "0.450438317792"),
              (621, 1366, 26, "0.481969000038"), (683, 1502, 27, "0.51570683004"), (751, 1652, 28, "0.551806308143"),
              (826, 1816, 29, "0.590432749713")]
    out = ["V -1 1 NFEAT 0"]
    for i, (cin, cout, kw, do) in enumerate(layers):
        out += [f"WN 3 C {cin} {cout} {kw} 1 {170 if i == 0 else 0}", "GLU 2", f"DO {do}"]
    out += ["RO 2 0 3 1", "WN 0 L 908 1816", "GLU 0", "DO 0.590432749713", "WN 0 L 908 NLABEL"]
    return "\n".join(out) + "\n"


def seq2seq_tds(ctc_head=True):
    out = ["V -1 NFEAT 1 0"]
    cin = 1
    for c, n in ((10, 2), (14, 3), (18, 6)):
        out += [f"C2 {cin} {c} 21 1 2 1 -1 -1", "R", "DO 0.2", "LN 3"] + [f"TDS {c} 21 80 0.2"] * n
        cin = c
    out += ["V 0 1440 1 0", "RO 1 0 3 2", "L 1440 NLABEL" if ctc_head else "L 1440 1024"]
    return "\n".join(out) + "\n"


def streaming_tds():
    # (channels, PD left, PD right, C2 kernel, C2 stride, TDS kernel, [right padding of each TDS block])
    stages = [(15, 5, 3, 10, 2, 9, [1, 1]), (19, 7, 1, 10, 2, 9, [1, 1, 1]), (23, 9, 1, 12, 2, 11, [1, 1, 1, 0]),
              (27, 10, 0, 11, 1, 11, [0, 0, 0, 0, 0])]
    out = ["V -1 NFEAT 1 0", "SAUG 80 27 2 100 1.0 2"]
    cin = 1
    for c, pl, pr, k, s, tk, rpads in stages:
        out += [f"PD 0 {pl} {pr}", f"C2 {cin} {c} {k} 1 {s} 1 0 0", "R", "DO 0.1", "LN 1 2"]
        out += [f"TDS {c} {tk} 80 0.1 0 {r} 0" for r in rpads]
        cin = c
    out += ["RO 2 1 0 3", "V 2160 -1 1 0", "L 2160 NLABEL", "V NLABEL 0 -1 1"]
    return "\n".join(out) + "\n"


def learnable_frontend_timit():
    """7 x (C2 over features-as-channels, kernel 5, SAME padding; PReLU; dropout 0.7), then the Linear head"""
    out = ["V -1 1 NFEAT 0"]
    cin = "NFEAT"
    for _ in range(7):
        out += [f"C2 {cin} 1000 5 1 1 1 -1 0", "PR", "DO 0.7"]
        cin = 1000
    out += ["RO 2 0 3 1", "L 1000 NLABEL"]
    return "\n".join(out) + "\n"


LEARNABLE_FRONTEND_FILE = "recipes/learnable_frontend/am_baseline_conv_relu.arch"


# BASELINE.json configs[i] -> (generator, criterion, filterbanks, default label count)
BASELINE_ARCHS = {
    "conv_glu_wsj": (conv_glu_wsj, "asg", 40, 30),
    "seq2seq_tds_ctc": (seq2seq_tds, "ctc", 80, 10000),
    "conv_glu_librispeech": (conv_glu_librispeech, "asg", 40, 30),
    "streaming_tds_ctc": (streaming_tds, "ctc", 80, 10000),
}
REFERENCE_FILES = {
    "conv_glu_wsj": "recipes/conv_glu/wsj/network.arch",
    "seq2seq_tds_ctc": "recipes/seq2seq_tds/librispeech/network.arch",
    "conv_glu_librispeech": "recipes/conv_glu/librispeech/network.arch",
    "streaming_tds_ctc": "recipes/streaming_convnets/librispeech/am_500ms_future_context.arch",
}
