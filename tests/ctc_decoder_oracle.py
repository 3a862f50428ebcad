"""numpy restatement of the CUDA CTC prefix beam search (models/decoder/_cuda_ctc_decoder.py, cuctc/).

float64 with exact log / exp, string prefixes (tuples) instead of a trie, and the kernel's tie rule: among equal keys
the lower ``beam * V + token`` wins, the stay entry counting as token 0.  ``oracle_beam`` keeps more beams than the
kernel can (to decode with nothing pruned); by default it is ``beam``.
"""
from __future__ import annotations

import numpy as np


def _lse(a, b):
    return np.logaddexp(a, b)


def decode(lp, length, beam, threshold, oracle_beam=None, stats=None):
    """Decode one row ``lp`` [T][V] over its first ``length`` frames; ``threshold`` is the log blank-skip threshold.

    Returns ``(hyps, margins)``: ``hyps`` a list of ``(tokens tuple, score)`` best first (``beam`` of them, or as many
    as there are beams), ``margins`` each step's gap between the ``beam``-th and ``(beam + 1)``-th keys (inf where there
    is no ``(beam + 1)``-th).  With a dict ``stats``, ``stats["recreated_merges"]`` counts the merges of a beam
    ``A + c`` into a beam ``B`` whose own parent was an earlier instance of ``A``'s prefix (one that left the beam and
    was re-created): the case where a trie must compare strings, not nodes.
    """
    lp = np.asarray(lp, dtype=np.float64)
    V = lp.shape[1]
    keep = oracle_beam or beam
    sel = [t for t in range(length) if lp[t, 0] < threshold]
    if not sel:
        return [], []
    margins = []

    def collapse(s):
        return s + 1 < len(sel) and sel[s + 1] - sel[s] > 1

    cur = lp[sel[0]]
    order = np.lexsort((np.arange(V), -cur))
    if keep < V:
        margins.append(cur[order[keep - 1]] - cur[order[keep]])
    else:
        margins.append(np.inf)
    beams = []  # (prefix, pb, pnb, score)
    inst = []  # (instance id of the prefix, instance id of its parent prefix)
    count = [0]

    def fresh():
        count[0] += 1
        return count[0]

    recreated = 0
    for c in order[:keep]:
        key = cur[c]
        inst.append((0, -1) if c == 0 else (fresh(), 0))
        if c == 0:
            beams.append(((), key, -np.inf, key))
        else:
            beams.append(((int(c),), key, -np.inf, key) if collapse(0) else ((int(c),), -np.inf, key, key))
    for s in range(1, len(sel)):
        cur = lp[sel[s]]
        nb = len(beams)
        pb = np.array([x[1] for x in beams])
        pnb = np.array([x[2] for x in beams])
        K = _lse(pb, pnb)
        # table[i][c]: stay at c = 0, extension by c otherwise, as (p_blank, p_nonblank)
        tb = np.full((nb, V), -np.inf)
        tn = cur[None, :] + K[:, None]
        tb[:, 0] = cur[0] + K
        tn[:, 0] = -np.inf
        for i, (p, b_, n_, _) in enumerate(beams):
            if p:
                tn[i, 0] = cur[p[-1]] + n_
                tn[i, p[-1]] = cur[p[-1]] + b_
        for i, (p, _, _, _) in enumerate(beams):  # merges: beam i extended by c is beam j
            for j, (q, _, _, _) in enumerate(beams):
                if len(q) == len(p) + 1 and q[:-1] == p:
                    recreated += inst[j][1] != inst[i][0]
                    c = q[-1]
                    tb[j, 0] = _lse(tb[j, 0], tb[i, c])
                    tn[j, 0] = _lse(tn[j, 0], tn[i, c])
                    tb[i, c] = tn[i, c] = -np.inf
        keys = _lse(tb, tn)
        merged = (tb == -np.inf) & (tn == -np.inf)
        keys[merged] = -np.inf
        flat = keys.ravel()
        if flat.size > 4 * (keep + 1):  # only the best keep + 1 matter (a tie there shows as a zero margin)
            part = np.argpartition(-flat, keep)[: keep + 1]
            order = part[np.lexsort((part, -flat[part]))]
        else:
            order = np.lexsort((np.arange(flat.size), -flat))
        live = int((flat > -np.inf).sum())
        take = min(keep, live)
        margins.append(flat[order[take - 1]] - flat[order[take]] if take < live else np.inf)
        col = collapse(s)
        new, new_inst = [], []
        for idx in order[:take]:
            i, c = divmod(int(idx), V)
            new_inst.append(inst[i] if c == 0 else (fresh(), inst[i][0]))
            p = beams[i][0] if c == 0 else beams[i][0] + (c,)
            key = flat[idx]
            new.append((p, key, -np.inf, key) if col else (p, tb[i, c], tn[i, c], key))
        beams, inst = new, new_inst
    if stats is not None:
        stats["recreated_merges"] = recreated
    return [(x[0], x[3]) for x in beams[:beam]], margins


def exact_prefix_scores(lp):
    """log P(prefix) for every collapsed label sequence, by enumerating all V^T alignments (tiny V and T only)."""
    lp = np.asarray(lp, dtype=np.float64)
    T, V = lp.shape
    out = {}
    for path in np.ndindex(*([V] * T)):
        s = sum(lp[t, c] for t, c in enumerate(path))
        seq, prev = [], 0
        for c in path:
            if c != 0 and c != prev:
                seq.append(c)
            prev = c
        k = tuple(seq)
        out[k] = np.logaddexp(out.get(k, -np.inf), s)
    return out
