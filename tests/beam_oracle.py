"""Float64 restatement of the engine's beam search (include/valle_b200.h "Beam search") over any AR logits function.

beam_search(logits_fn, n, cap_new) runs the search of one utterance: logits_fn(tokens) returns the float64 [1025] AR
logits after the generated first-codebook ids `tokens` (a list).  Scores are float64 sums of l - logsumexp(l).  Beside
the result it returns the smallest margin of every decision the search took, so that a caller can keep only cases an
fp32 search must decide the same way:
  * the selection: the score gap between the n-th and the (n+1)-th non-EOS candidate (which hypotheses survive);
  * each EOS candidate near the top: its gap to the n-th best of the other candidates (whether it ranks below n);
  * the finished hypothesis: the gap of an offered EOS candidate to it, of it to the best live beam (the stop rule)
    and, at the cap, of it to beam 0.
"""
from __future__ import annotations

import math

import torch

EOS = 1024


def beam_search(logits_fn, n: int, cap_new: int, tok_stride: int = 1 << 30):
    """-> (tokens of the winner, its score over its codes, smallest decision margin, 'eos' or 'cap')"""
    beams = [([], 0.0)] + [None] * (n - 1)      # (tokens, score); None: score -inf (only beam 0 starts)
    fin = None                                   # (tokens, ranking score c, score over the codes)
    margin = math.inf
    t = 0
    while True:
        if t > cap_new or t >= tok_stride:
            if fin is not None:
                margin = min(margin, abs(fin[1] - beams[0][1]))
                if fin[1] >= beams[0][1]:
                    return fin[0], fin[2], margin, "cap"
            return beams[0][0], beams[0][1], margin, "cap"
        cands = []                               # (c, l, j, v)
        for j, b in enumerate(beams):
            if b is None:
                continue
            l = logits_fn(b[0]).double()
            inc = (l - torch.logsumexp(l, 0)).tolist()
            lv = l.tolist()
            cands += [(b[1] + inc[v], lv[v], j, v) for v in range(len(lv))]
        cands.sort(key=lambda c: (-c[0], -c[1], c[2], c[3]))
        top = cands[:2 * n + 2]
        non_eos = [c for c in top if c[3] != EOS]
        margin = min(margin, non_eos[n - 1][0] - non_eos[n][0])
        for r, c in enumerate(top):
            if c[3] == EOS:
                others = [o for o in top if o is not c]
                margin = min(margin, abs(c[0] - others[n - 1][0]))
                if r < n:
                    if fin is not None:
                        margin = min(margin, abs(c[0] - fin[1]))
                    if fin is None or c[0] > fin[1]:
                        fin = (list(beams[c[2]][0]), c[0], beams[c[2]][1])
        beams = [(beams[c[2]][0] + [c[3]], c[0]) for c in non_eos[:n]]
        t += 1
        if fin is not None:
            margin = min(margin, abs(fin[1] - beams[0][1]))
            if fin[1] >= beams[0][1]:
                return fin[0], fin[2], margin, "eos"
