"""Plain-Python model of the device scoring contract (csrc/text_eval.cu, DESIGN.md §10): the token tables
w2l_text_device_create builds, the table-driven path -> letters -> words transform, the word ids and the Levenshtein
programme with EditDistanceMeter's tie order.  tests/test_eval_cpu.py pins it against the host pipeline; the GPU tests
compare the kernels with the host pipeline directly."""
from __future__ import annotations

import random

# the vocabularies the tests draw from: plain letters, multi-byte UTF-8 letters, and multi-letter tokens
LETTER_TOKENS = ["|", "'", "a", "b", "c", "é", "ß", "中", "ab"]
WORDPIECE_TOKENS = ["_a", "b", "_bé", "中", "_", "ab", "a", "_中ß", "|"]


class Tables:
    """token roles, letters and letter bytes of one pipeline, as w2l_text_device_create builds them"""

    def __init__(self, tokens, criterion="ctc", replabel=0, surround="", wordpiece=False, wordsep="|"):
        entries = list(tokens) + [f"<{r}>" for r in range(1, replabel + 1)]
        if criterion == "ctc":
            entries.append("#")
        if criterion == "seq2seq":
            entries += ["$", "<pad>"]
        idx = {e: i for i, e in enumerate(entries)}
        self.N, self.criterion, self.replabel = len(entries), criterion, replabel
        self.role = [0] * self.N
        for r in range(1, replabel + 1):
            self.role[idx[f"<{r}>"]] = r
        self.blank = idx["#"] if criterion == "ctc" else -1
        self.eos = idx["$"] if criterion == "seq2seq" else -1
        self.pad = idx["<pad>"] if criterion == "seq2seq" else -1
        self.sil = idx.get("|", -1)
        self.surround = idx[surround] if surround else -1
        self.letters: list[str] = []
        ids: dict[str, int] = {}
        self.spell = []
        for e in entries:
            row = []
            for s in (list(e) if wordpiece else [e]):  # a str's characters are splitWrd's code points
                if s not in ids:
                    ids[s] = len(self.letters)
                    self.letters.append(s)
                row.append(ids[s])
            self.spell.append(row)
        self.sep = ids.get(wordsep, -1) if wordsep else -1


def words_of(t: Tables, row, hyp: bool):
    """(letters, words as lists of letter ids) of a hypothesis (tknPrediction2Ltr) or target (tknTarget2Ltr) row, or
    None where the host throws"""
    row = [int(v) for v in row]
    s2s = t.criterion == "seq2seq"
    if hyp:
        if s2s and t.eos in row:
            row = row[: row.index(t.eos)]
        toks = []
        for i, v in enumerate(row):
            keep = not (s2s and v == t.pad)
            if t.criterion in ("ctc", "asg") and i > 0 and row[i - 1] == v:
                keep = False
            if t.criterion == "ctc" and v == t.blank:
                keep = False
            if v == -1:
                keep = False
            if keep:
                toks.append(v)
    else:
        n = len(row)
        while n > 0 and row[n - 1] < 0:
            n -= 1
        toks = [v for v in row[:n] if not (s2s and v == t.pad)]
    if s2s:
        while toks and toks[-1] == t.eos:
            toks.pop()

    def role(v):
        return t.role[v] if 0 <= v < t.N else 0

    if t.replabel > 0:
        out = []
        for i, v in enumerate(toks):
            r = role(v)
            if r == 0:
                out.append(v)
            elif i > 0 and role(toks[i - 1]) == 0:
                out += [toks[i - 1]] * r
        toks = out
    for tr in (t.sil, t.surround):
        if tr >= 0:
            if toks and toks[-1] == tr:
                toks.pop()
            if toks and toks[0] == tr:
                toks.pop(0)
    if any(not 0 <= v < t.N for v in toks):
        return None
    letters = [l for v in toks for l in t.spell[v]]
    if t.sep >= 0:
        if letters and letters[0] == t.sep:
            letters.pop(0)
        if letters and letters[-1] == t.sep:
            letters.pop()
    words, cur = [], []
    for l in letters:
        if l == t.sep:
            if cur:
                words.append(cur)
            cur = []
        else:
            cur.append(l)
    if cur:
        words.append(cur)
    return letters, words


def word_ids(t: Tables, hyp_words, ref_words):
    """a reference word -> the index of the first equal reference word; a hypothesis word -> the index of the first
    equal reference word, else -1 - its own index.  Equal = the same string (bytes), as tkn2Wrd's words compare."""
    key = [("".join(t.letters[l] for l in w)).encode() for w in ref_words]
    rid = [key.index(k) for k in key]
    hid = []
    for k, w in enumerate(hyp_words):
        s = "".join(t.letters[l] for l in w).encode()
        hid.append(key.index(s) if s in key else -1 - k)
    return hid, rid


def edit(hyp, ref):
    """(ndel, nins, nsub) of EditDistanceMeter::levensteinDistance: per cell substitution / match, then deletion, then
    insertion, each taken only with a strictly smaller sum"""
    prev = [(j, 0, 0) for j in range(len(ref) + 1)]
    for i in range(1, len(hyp) + 1):
        cur = [(0, i, 0)]
        for j in range(1, len(ref) + 1):
            s = prev[j - 1]
            best = (s[0], s[1], s[2] + (hyp[i - 1] != ref[j - 1]))
            d = cur[j - 1]
            d = (d[0] + 1, d[1], d[2])
            if sum(d) < sum(best):
                best = d
            n = prev[j]
            n = (n[0], n[1] + 1, n[2])
            if sum(n) < sum(best):
                best = n
            cur.append(best)
        prev = cur
    return prev[-1]


def counts(t: Tables, path, target, path_length=None):
    """the eight counts of one utterance: reference letters, del, ins, sub, then the same for words; -1s where the host
    throws"""
    if path_length is not None:
        if not 0 <= path_length <= len(path):
            return [-1] * 8
        path = path[:path_length]
    h, r = words_of(t, path, True), words_of(t, target, False)
    if h is None or r is None:
        return [-1] * 8
    hid, rid = word_ids(t, h[1], r[1])
    return [len(r[0]), *edit(h[0], r[0]), len(r[1]), *edit(hid, rid)]


# ---- random cases ---------------------------------------------------------------------------------------------------
def pipeline_args(criterion, replabel, surround, wordpiece):
    tokens = WORDPIECE_TOKENS if wordpiece else LETTER_TOKENS
    return dict(tokens=tokens, criterion=criterion, replabel=replabel, surround=surround, wordpiece=wordpiece,
                wordsep="_" if wordpiece else "|")


def random_row(rng: random.Random, t: Tables, n: int, hyp: bool, invalid_rate=0.003, minus_one=0.03):
    """a row with runs (so uniq and replabels matter), specials, -1 and pad inside, and rarely a token outside [0, N)"""
    specials = [v for v in (t.blank, t.eos, t.pad, t.sil, t.surround) if v >= 0] + [i for i, r in enumerate(t.role) if r > 0]
    row = []
    while len(row) < n:
        u = rng.random()
        if u < invalid_rate:
            v = rng.choice([t.N, t.N + 5, -2])
        elif u < invalid_rate + minus_one:
            v = -1
        elif u < 0.3 and specials:
            v = rng.choice(specials)
        else:
            v = rng.randrange(t.N)
        row += [v] * rng.choice([1, 1, 1, 2, 3])
    row = row[:n]
    if not hyp and rng.random() < 0.5:  # trailing padding
        k = rng.randrange(0, n + 1)
        row[k:] = [t.pad if t.criterion == "seq2seq" else -1] * (n - k)
    return row
