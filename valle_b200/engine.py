"""Batched VALL-E decoding engine: the host side of the hot path.

Implements the loops of `VALLE.inference` (valle/models/valle.py:961-1137) for B independent
utterances at once on one GPU:

  * AR: ragged prefill of text + acoustic prompt (fills the KV cache), then single-row decode
    steps against the growing KV cache (the reference recomputes the whole sequence per token,
    valle.py:1004 TODO).  The KV cache is exact under the reference's mask: text rows attend to
    text only, audio rows to text + causal audio (valle.py:1019-1030), so cached K/V never change.
    All loop state (lengths, tokens, stop flags) lives on the device; a decode step is one CUDA
    graph replay; the host only polls the stop flags every `poll` steps (the reference does a
    D2H sync + an H2D mask copy per token).
  * NAR: 7 full-attention passes over packed [text | prompt | generated] rows with AdaLN stage
    conditioning, argmax and the embedding accumulation fused on the device (valle.py:1115-1134).

torch is used for allocation, streams and index bookkeeping; all arithmetic runs in
libvalle_b200.so.  There is no CPU fallback.
"""
from __future__ import annotations

import math
import os

import ctypes as C
from dataclasses import dataclass
from typing import Dict, Iterable, Iterator, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L
from . import ops

NUM_AUDIO_TOKENS = 1024  # valle/models/macros.py:5
NUM_TEXT_TOKENS = 512    # valle/models/macros.py:2


def _on_device(fn):
    """Run a method with the engine's GPU as the current CUDA device: every kernel launch, stream and event of the
    call then belongs to `self.device` even when the caller's current device is another GPU of the box."""
    import functools

    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        with torch.cuda.device(self.device):
            return fn(self, *args, **kwargs)
    return wrapper


def _check_utt(who: str, text: torch.Tensor, codes: torch.Tensor, Q: int, name: str = "prompt code"):
    """One utterance's inputs: text [S > 0] phoneme ids and codes [T, Q] codec ids (the prompt, or continual()'s
    codes); ValueError for a shape.  nn.Embedding raises IndexError for ids outside the table
    (valle/modules/embedding.py:46): host tensors are checked here before the copy, device tensors by the kernels
    (clamped read + flag, ops.check_oob).  The first codebook's tables have 1025 rows (+ <BOS>)."""
    if text.ndim != 1 or text.numel() == 0 or codes.ndim != 2 or codes.shape[1] != Q:
        raise ValueError(f"{who}: expected text ids [S > 0] and {name}s [T, {Q}]")
    for t, hi, what in ((text, NUM_TEXT_TOKENS, "phoneme"),
                        (codes[:, :1], NUM_AUDIO_TOKENS + 1, f"{name} (first codebook)"),
                        (codes[:, 1:], NUM_AUDIO_TOKENS, name)):
        if not t.is_cuda and t.numel() > 0:
            lo_v, hi_v = int(t.min()), int(t.max())
            if lo_v < 0 or hi_v >= hi:
                raise IndexError(f"index out of range in self: {what} id {lo_v if lo_v < 0 else hi_v} not in [0, {hi})")


@dataclass
class EngineStats:
    """CUDA-event timings (ms) of the phases of the last generate() / generate_stream() call and the number of decode
    steps; generate_stream() also counts the requests it admitted into decode slots and the decode steps their
    candidates ran, a beam group's rows counted each (slot occupancy = slot_steps / (ar_steps * slots))"""
    ar_steps: int = 0
    ar_ms: float = 0.0
    prefill_ms: float = 0.0
    nar_ms: float = 0.0
    admissions: int = 0
    slot_steps: int = 0


class StreamRequest(NamedTuple):
    """One utterance of ValleEngine.generate_stream: text int64 [S] phoneme ids, prompt int64 [Tp, Q] codec ids, and
    what generate() takes per utterance.  top_k != 1 and ras need a seed (the seeded device sampler); num_beams > 1
    decodes it by beam search, as generate(num_beams=) does, and takes no seed, top_k, top_p or ras."""
    text: torch.Tensor
    prompt: torch.Tensor
    enroll_len: Optional[int] = None
    seed: Optional[int] = None
    top_k: int = 1
    temperature: float = 1.0
    max_new_tokens: Optional[int] = None
    top_p: float = 1.0
    ras: Optional[Tuple[int, float]] = None
    num_beams: int = 1


class BestOfRequest(NamedTuple):
    """A best-of-n request of ValleEngine.generate_stream: `request` (a StreamRequest, or a tuple in its field order, with
    a seed s and num_beams == 1) decoded as num_samples candidates, candidate j drawing from seed s + j with the
    request's top_k / temperature / top_p / ras / max_new_tokens, as generate([text], [prompt], seed=s,
    num_samples=n) draws them.  It yields the n candidates' codes as a list; num_samples == 1 is the plain request."""
    request: StreamRequest
    num_samples: int


def _as_request(r):
    """an item of generate_stream's requests: a BestOfRequest (its request coerced), or a StreamRequest / a tuple in
    its field order.  BestOfRequest is a tuple too, so it is recognised first."""
    if isinstance(r, BestOfRequest):
        return BestOfRequest(StreamRequest(*r.request), r.num_samples)
    return StreamRequest(*r)


class _Candidates:
    """The candidates of one request in the stream as they decode and come back from the NAR: n rows of a best-of
    request, or the one utterance of a plain or beam request.  parent: the slot a best-of request was prefilled into,
    whose cache holds the prompt prefix its other candidates read (kv_parent); it stays held until every candidate has
    stopped.  None: each candidate's slot is freed when it stops."""

    def __init__(self, index: int, n: int, parent: Optional[int] = None, best_of: bool = False, beam: bool = False):
        self.index, self.parent, self.best_of, self.beam = index, parent, best_of, beam
        self.running = set()            # slots of the candidates still decoding
        self.codes: List[Optional[torch.Tensor]] = [None] * n
        self.scores: List[Optional[torch.Tensor]] = [None] * n
        self.left = n                   # candidates not back from the NAR yet

    def stop(self, slot: int) -> List[int]:
        """the slots freed when the candidate in `slot` stops: its own, except the parent while a candidate still reads
        it, and the parent with the last candidate"""
        self.running.discard(slot)
        freed = [] if slot == self.parent else [slot]
        if self.parent is not None and not self.running:
            freed.append(self.parent)
        return freed

    def done(self, j: int, codes: torch.Tensor, score: Optional[torch.Tensor]) -> bool:
        """candidate j's codes (and score) from the NAR; True once every candidate is back"""
        self.codes[j], self.scores[j] = codes, score
        self.left -= 1
        return self.left == 0

    def result(self, scores: bool) -> tuple:
        """(index, codes) or (index, codes, scores): a best-of request's n codes and scores [n], a plain request's codes
        and scores [1], a beam request's codes and its winner's score (0-d)"""
        codes = self.codes if self.best_of else self.codes[0]
        if not scores:
            return self.index, codes
        sc = torch.stack(self.scores) if self.best_of else self.scores[0] if self.beam else self.scores[0].view(1)
        return self.index, codes, sc


def _take_slots(free: List[int], widths: Sequence[int]) -> List[List[int]]:
    """First-in first-out admission into decode slots.  widths: the slots each queued request needs, in queue order (1,
    n for a beam group of n rows, or n for the n candidates of a best-of request).  Each request takes the lowest run
    of that many consecutive free slots, up to the first request that finds no such run: it waits, and every request
    behind it waits too.  free: the free slots,
    sorted; the taken ones are removed from it.  Returns the slots of the requests that were admitted."""
    out = []
    for n in widths:
        i = next((i for i in range(len(free) - n + 1) if free[i + n - 1] == free[i] + n - 1), None)
        if i is None:
            break
        out.append(free[i:i + n])
        del free[i:i + n]
    return out


def _stream_draws(idx: int, item, Q: int, n_slots: int, fp8: bool) -> Tuple[StreamRequest, List[_Draw]]:
    """Request `idx` of generate_stream (a StreamRequest or a BestOfRequest, coerced), validated as generate() would
    validate it alone, plus n <= n_slots: the request, its num_beams an int, and the draws of its candidates (one for
    a plain or beam request, n for a best-of request: seeds s + j).  ValueError names the request."""
    r, n = (item.request, item.num_samples) if isinstance(item, BestOfRequest) else (item, 1)
    _check_utt(f"request {idx}", r.text, r.prompt, Q)
    try:
        beams = _check_num_beams(r.num_beams, r.seed, r.top_k, r.top_p, r.ras, n, None, None, False, fp8)
        n = _check_num_samples(n, r.seed, False, None, None, False, None)
    except ValueError as e:
        raise ValueError(f"request {idx}: {e}") from None
    if beams > n_slots:
        raise ValueError(f"request {idx}: num_beams={beams} needs more than the {n_slots} slots")
    if n > n_slots:
        raise ValueError(f"request {idx}: num_samples={n} needs more than the {n_slots} slots")
    seed, top_k = r.seed, r.top_k
    if seed is None:
        if top_k != 1 or r.ras is not None:
            raise ValueError(f"request {idx}: top_k={top_k} / ras need a seed (the seeded device sampler)")
        seed = 0
    draws = _draws(n, seed, top_k, r.temperature, r.top_p, None if r.ras is None else [r.ras] * n)
    return r._replace(num_beams=beams), draws


class _ArBuffers:
    """Persistent device state for the AR loop at one (B, cache_cap, tok_stride, cache dtype) shape, plus the CUDA
    graphs of decode steps captured on it.  kv_dtype torch.float8_e4m3fn: the FP8 cache (e4m3 rows and one exponent
    byte per cached row, include/valle_b200.h "FP8 (e4m3) KV cache"); None: the engine dtype."""

    def __init__(self, eng: "ValleEngine", B: int, cap: int, tok_stride: int, kv_dtype: Optional[torch.dtype] = None):
        dev, d = eng.device, eng.d
        nd = eng.ar
        self.B, self.cap, self.tok_stride, self.kv_dtype = B, cap, tok_stride, kv_dtype
        i32 = dict(dtype=torch.int32, device=dev)
        self.text_len = torch.zeros(B, **i32)
        self.prompt_len = torch.zeros(B, **i32)
        self.max_new = torch.zeros(B, **i32)
        self.n_gen = torch.zeros(B, **i32)
        self.finished = torch.zeros(B, **i32)
        self.tokens = torch.zeros((B, tok_stride), **i32)
        self.x_cur = torch.zeros((B, d), dtype=torch.float32, device=dev)
        self.ldl = (eng.n_vocab + 3) // 4 * 4
        self.logits = torch.zeros((B, self.ldl), dtype=torch.float32, device=dev)
        self.kcache = torch.zeros((nd.n_layer, B, nd.H, cap, 64), dtype=kv_dtype or eng.dtype, device=dev)
        self.vcache = torch.zeros_like(self.kcache)
        fp8 = kv_dtype == torch.float8_e4m3fn
        #: FP8 cache: the biased exponent (e + 127) of every cached row, [n_layer, B, H, cap] uint8
        self.k_exp = torch.zeros((nd.n_layer, B, nd.H, cap), dtype=torch.uint8, device=dev) if fp8 else None
        self.v_exp = torch.zeros_like(self.k_exp) if fp8 else None
        # seeded device sampler, per row (uint64 seeds stored as their int64 bit patterns)
        self.sample_seed = torch.zeros(B, dtype=torch.int64, device=dev)
        self.top_k = torch.zeros(B, **i32)
        self.temperature = torch.ones(B, dtype=torch.float32, device=dev)
        self.top_p = torch.ones(B, dtype=torch.float32, device=dev)
        self.ras_window = torch.zeros(B, **i32)
        self.ras_max = torch.zeros(B, **i32)
        #: best-of-n: each row's parent row (the shared prompt prefix of its cache) and its AR log-likelihood; the
        #: state points at them only in calls that use them (set_best_of)
        self.kv_parent = torch.zeros(B, **i32)
        self.logprob = torch.zeros(B, dtype=torch.float32, device=dev)
        #: beam search (include/valle_b200.h "Beam search"): each row's ancestry and score, and each group's finished
        #: hypothesis (rows [0, B / n) of the fin arrays); the state points at them only in beam calls (set_best_of)
        self.beam_anc = torch.zeros((B, tok_stride), dtype=torch.uint8, device=dev)
        self.beam_score = torch.zeros(B, dtype=torch.float32, device=dev)
        self.beam_fin_score = torch.zeros((B, 2), dtype=torch.float32, device=dev)
        self.beam_fin_len = torch.zeros(B, **i32)
        self.beam_fin_anc = torch.zeros((B, tok_stride), dtype=torch.uint8, device=dev)
        #: per-row beam groups of continuous batching (set_groups): each row's group's first row (-1: none), its width
        self.beam_first = torch.full((B,), -1, **i32)
        self.beam_n = torch.zeros(B, **i32)
        st = L.ArState()
        st.B, st.tok_stride = B, tok_stride
        st.text_len, st.prompt_len, st.max_new = self.text_len.data_ptr(), self.prompt_len.data_ptr(), self.max_new.data_ptr()
        st.n_gen, st.finished, st.tokens = self.n_gen.data_ptr(), self.finished.data_ptr(), self.tokens.data_ptr()
        st.x_cur, st.logits = self.x_cur.data_ptr(), self.logits.data_ptr()
        st.kcache, st.vcache = self.kcache.data_ptr(), self.vcache.data_ptr()
        st.cache_layer_stride, st.cache_seq_stride, st.cache_cap = self.kcache.stride(0), self.kcache.stride(1), cap
        st.sample_seed, st.top_k = self.sample_seed.data_ptr(), self.top_k.data_ptr()
        st.temperature = self.temperature.data_ptr()
        st.top_p, st.ras_window, st.ras_max = self.top_p.data_ptr(), self.ras_window.data_ptr(), self.ras_max.data_ptr()
        if fp8:
            st.kv_dtype, st.k_exp, st.v_exp = L.VB_E4M3, self.k_exp.data_ptr(), self.v_exp.data_ptr()
        self.st = st
        nbytes = eng.lib.vb_ar_step_workspace(C.byref(nd.desc), B, cap)
        self.ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        #: (head tables, draw mode, steps) -> (graph of that many decode steps, kernels per replay, head struct)
        self.graphs: Dict[tuple, Tuple[torch.cuda.CUDAGraph, int, L.ArHead]] = {}
        self.eng = eng

    def set_best_of(self, n_rows: int, n: int, scores: bool, beams: bool = False):
        """Point the state at kv_parent when n > 1 (row r of the first n_rows reads its parent r - r % n's prompt
        prefix) and at logprob, zeroed, with scores; leave either NULL otherwise.  The FP8 cache keeps kv_parent NULL:
        there the shared read is slower than every row reading its own copy (DESIGN section 7), and the codes are
        the same either way.  beams: the rows are groups of n beams (beam search), whose arrays the state then points
        at, set to their starting values; otherwise beam search is off."""
        st = self.st
        st.beam_width, st.beam_anc, st.beam_score, st.beam_fin_score, st.beam_fin_len, st.beam_fin_anc = \
            0, None, None, None, None, None
        st.beam_first = st.beam_n = None
        if beams:
            r = torch.arange(n_rows, device=self.beam_score.device)
            self.beam_score[:n_rows] = torch.where(r % n == 0, 0.0, float("-inf"))
            self.beam_fin_score[:, 0] = float("-inf")
            st.beam_width = n
            self._point_beams()
        self.st.kv_parent = None
        if n > 1 and self.kv_dtype is None:
            r = torch.arange(n_rows, dtype=torch.int32)
            self.kv_parent[:n_rows].copy_(r - r % n)
            self.st.kv_parent = self.kv_parent.data_ptr()
        self.st.logprob = None
        if scores:
            self.logprob.zero_()
            self.st.logprob = self.logprob.data_ptr()

    def _point_beams(self):
        st = self.st
        st.beam_anc, st.beam_score = self.beam_anc.data_ptr(), self.beam_score.data_ptr()
        st.beam_fin_score, st.beam_fin_len = self.beam_fin_score.data_ptr(), self.beam_fin_len.data_ptr()
        st.beam_fin_anc = self.beam_fin_anc.data_ptr()

    def set_parents(self):
        """Point the state at kv_parent, every row its own parent (the stream sets a best-of request's rows to their
        parent when it admits them)"""
        self.kv_parent.copy_(torch.arange(self.B, dtype=torch.int32))
        self.st.kv_parent = self.kv_parent.data_ptr()

    def set_groups(self, parents: bool = True):
        """Point the state at per-row beam groups (vb_ar_state.beam_first, the stream's mixed head), every row in no
        group, and at kv_parent, every row its own parent (parents=False: keep the kv_parent table the state points at
        already); vb_ar_admit starts each group it admits"""
        self.beam_first.fill_(-1)
        if parents:
            self.set_parents()
        st = self.st
        st.beam_first, st.beam_n = self.beam_first.data_ptr(), self.beam_n.data_ptr()
        self._point_beams()

    def load_rows(self, p: _Prefill, draws: Optional[Sequence[_Draw]] = None,
                  groups: Optional[Sequence[Tuple[int, int, int]]] = None, parents: Optional[Sequence[int]] = None):
        """Write the lengths and token caps of prefill block p's utterances into their rows (0..B-1, or p.slots_d, and
        the rows forked from them, p.admit_d) and, given their draws, the sampler columns, all six from one host ->
        device copy; groups: also each row's (kv_parent, beam_first, beam_n) (set_groups), parents: its kv_parent
        alone (set_parents), in the same copy"""
        rows = None if p.slots_d is None else (p.slots_d if p.admit_d is None else p.admit_d).long()

        def put(col, v):
            if rows is None:
                col[:len(p.S)].copy_(v)
            else:
                col.index_copy_(0, rows, v)
        for col, v in ((self.text_len, p.S_d), (self.prompt_len, p.Tp_d), (self.max_new, p.capn_d)):
            put(col, v if p.gather_d is None else v.index_select(0, p.gather_d))
        if draws is None:
            return
        # _Draw's fields in order; the int64 seeds first, so that every column starts aligned to its element size
        cols = [self.sample_seed, self.top_k, self.temperature, self.top_p, self.ras_window, self.ras_max]
        vals = list(zip(*(d._replace(seed=d.seed_i64) for d in draws)))
        if groups is not None:
            cols += [self.kv_parent, self.beam_first, self.beam_n]
            vals += list(zip(*groups))
        elif parents is not None:
            cols.append(self.kv_parent)
            vals.append(tuple(parents))
        block = torch.cat([torch.tensor(v, dtype=c.dtype).view(torch.uint8) for c, v in zip(cols, vals)])
        block = block.to(self.text_len.device, non_blocking=True).split([len(draws) * c.element_size() for c in cols])
        for c, v in zip(cols, block):
            put(c, v.view(c.dtype))


class _Utt(NamedTuple):
    """One utterance on its way to the NAR: its index in the call, device text ids [S] and prompt codes [Tp, Q], the
    prompt length the AR saw (Tp + 1 with <BOS>), and the enrolled phonemes the NAR text leaves out in prefix modes
    2 / 4 (None: the whole text)"""
    index: int
    text: torch.Tensor
    prompt: torch.Tensor
    Tp_ar: int
    enroll_len: Optional[int] = None


class _Prefill(NamedTuple):
    """The device-side inputs of one packed AR prefill of B utterances (ValleEngine._prefill_inputs)"""
    S: List[int]                    # text lengths
    Tp: List[int]                   # prompt lengths the AR sees (+1 for <BOS> with prepend_bos)
    Tp_nar: List[int]               # prompt lengths the NAR sees
    text_all: torch.Tensor          # int64 [sum S] phoneme ids
    prm_all: torch.Tensor           # int64 [sum Tp_nar, Q] prompt codes
    ar_tok: Optional[torch.Tensor]  # prepend_bos: int64 [sum Tp], <BOS> and the first codebook of every prompt
    # int32 views of one device block: the packed layout (cu_seqlens, lengths, rows / positions of the text and
    # prompt rows, the last row of every utterance), the token caps and the decode slots (None: rows 0..B-1)
    cu_d: torch.Tensor
    S_d: torch.Tensor
    Tp_d: torch.Tensor
    capn_d: torch.Tensor
    trow_d: torch.Tensor
    tpos_d: torch.Tensor
    arow_d: torch.Tensor
    apos_d: torch.Tensor
    last_d: torch.Tensor
    slots_d: Optional[torch.Tensor]
    # rows admitted next to the prefilled ones that take an utterance's prefill (vb_ar_fork_prefix): every admitted
    # row's slot, slots_d's then the forked rows', and the utterance each takes its lengths and last prefill row from
    admit_d: Optional[torch.Tensor] = None
    gather_d: Optional[torch.Tensor] = None

    def utts(self, index: Sequence[int], enroll_lens: Sequence[Optional[int]]) -> List[_Utt]:
        return [_Utt(i, t, pr, tp, None if e is None else int(e)) for i, t, pr, tp, e in
                zip(index, self.text_all.split(self.S), self.prm_all.split(self.Tp_nar), self.Tp, enroll_lens)]


def _is_seq(v) -> bool:
    return isinstance(v, (list, tuple)) or (isinstance(v, (torch.Tensor, np.ndarray)) and v.ndim > 0)


def _offsets(lens) -> np.ndarray:
    """[0, l0, l0 + l1, ..., sum]: where each ragged segment starts, then the total (int64)"""
    return np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).astype(np.int64)


def _check_top_p(ps):
    if any(not 0.0 < p <= 1.0 for p in ps):   # NaN fails too
        raise ValueError("top_p must lie in (0, 1]")


class _Draw(NamedTuple):
    """One utterance's seeded device draw, the sampler columns of vb_ar_state: top-k, temperature and top-p, then
    repetition-aware sampling over the last ras_window codes (0: off), which draws again when the draw occurs there
    more than ras_max times"""
    seed: int
    top_k: int
    temperature: float
    top_p: float
    ras_window: int
    ras_max: int

    @property
    def greedy(self) -> bool:
        """argmax: the seed draws nothing"""
        return self.top_k == 1 and self.ras_window == 0

    @property
    def seed_i64(self) -> int:
        """the uint64 seed as the int64 bit pattern the device column holds"""
        return self.seed - (1 << 64) if self.seed >= 1 << 63 else self.seed


def _ras_arrays(rows) -> Tuple[List[int], List[int]]:
    """(ras_window, ras_max) of validated (window K, threshold t) pairs / Nones (off): ras_max = floor(t K), the largest
    count c with c / K <= t, so that the device's integer test count > ras_max is exactly count / K > t as Python
    evaluates it (t K rounded to a double can land just below an integer: 0.29 * 100 = 28.999...)"""
    def ras_max(K, t):
        c = math.floor(t * K)
        while (c + 1) / K <= t:
            c += 1
        while c > 0 and c / K > t:
            c -= 1
        return c
    return [0 if r is None else r[0] for r in rows], [0 if r is None else ras_max(*r) for r in rows]


def _draws(B: int, seed, top_k, temperature, top_p=1.0, ras=None) -> List[_Draw]:
    """Validated draws of the B utterances of a seeded call.  An int seed s stands for s, s+1, ..., s+B-1 (so utterance
    b decoded alone with seed s+b draws what it draws in the batch), or B seeds, each in [0, 2**64); top_k /
    temperature / top_p: one value or a sequence of B; ras (repetition-aware sampling): None (off), one (window,
    threshold) pair for every utterance, or a sequence of B pairs / Nones, window an int in [1, 256], threshold in
    [0, 1)."""
    def per_row(v, what):
        if _is_seq(v):
            v = [x.item() if hasattr(x, "item") else x for x in v]
            if len(v) != B:
                raise ValueError(f"{what}: {len(v)} values for {B} utterances")
            return v
        return [v] * B
    if _is_seq(seed):
        seeds = per_row(seed, "seed")
    else:
        seeds = [int(seed) + b for b in range(B)]
    seeds = [int(x) for x in seeds]
    if any(x < 0 or x >= 1 << 64 for x in seeds):
        raise ValueError("seed: every utterance's seed must lie in [0, 2**64)")
    ks = [int(x) for x in per_row(top_k, "top_k")]
    ts = [float(x) for x in per_row(temperature, "temperature")]
    if any(not math.isfinite(t) or t <= 0.0 for t in ts):
        raise ValueError("temperature must be finite and > 0")
    ps = [float(x) for x in per_row(top_p, "top_p")]
    _check_top_p(ps)
    per = _is_seq(ras) and len(ras) > 0 and (ras[0] is None or _is_seq(ras[0]))
    rr = list(ras) if per else [ras] * B
    if len(rr) != B:
        raise ValueError(f"ras: {len(rr)} values for {B} utterances")
    for i, r in enumerate(rr):
        if r is not None:
            if not _is_seq(r) or len(r) != 2:
                raise ValueError(f"ras: expected a (window, threshold) pair, got {r!r}")
            w, t = r
            if isinstance(w, bool) or not isinstance(w, (int, np.integer)) or not 1 <= int(w) <= 256:
                raise ValueError(f"ras: the window must be an int in [1, 256] (got {w!r})")
            t = float(t)
            if not 0.0 <= t < 1.0:
                raise ValueError(f"ras: the threshold must lie in [0, 1) (got {t!r})")
            rr[i] = (int(w), t)
    return [_Draw(*v) for v in zip(seeds, ks, ts, ps, *_ras_arrays(rr))]


def _check_num_samples(n, seed, return_scores: bool, trace, forced, sample_on_host: bool, bf16_rows: Optional[int]):
    """Validated best-of-n arguments of generate(): n, an int >= 1.  n > 1 and return_scores need a seed (the seeded
    device sampler); n > 1 excludes the trace / forced test hooks; bf16_rows: the rows of one bf16 decode group, which
    must hold all n candidates of an utterance (None: no limit)"""
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 1:
        raise ValueError(f"num_samples must be an int >= 1 (got {n!r})")
    n = int(n)
    if (n > 1 or return_scores) and seed is None:
        raise ValueError("num_samples > 1 and return_scores need seed= (the seeded device sampler)")
    if (n > 1 or return_scores) and sample_on_host:
        raise ValueError("num_samples > 1 and return_scores draw on the device; they cannot be combined with "
                         "sample_on_host = True")
    if n > 1 and (trace is not None or forced is not None):
        raise ValueError("num_samples > 1 cannot be combined with the trace / forced test hooks")
    if return_scores and forced is not None:
        raise ValueError("return_scores scores the seeded draws; forced ids replace them")
    if bf16_rows is not None and n > bf16_rows:
        raise ValueError(f"num_samples={n}: a bf16 decode group holds at most {bf16_rows} candidates of one utterance")
    return n


def _check_num_beams(n, seed, top_k, top_p, ras, num_samples, trace, forced, sample_on_host: bool, fp8: bool) -> int:
    """Validated beam width of generate(): an int in [1, 16].  n > 1 searches by the AR log-likelihood alone, so it
    excludes every sampler argument (seed, top_k != 1, top_p, ras), best-of-n, host sampling, the trace / forced test
    hooks and the FP8 KV cache."""
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or not 1 <= n <= 16:
        raise ValueError(f"num_beams must be an int in [1, 16] (got {n!r})")
    n = int(n)
    if n == 1:
        return n
    if seed is not None or ras is not None or (_is_seq(top_k) or int(top_k) != 1) or \
            (_is_seq(top_p) or float(top_p) != 1.0):
        raise ValueError("num_beams > 1 ranks by the AR log-likelihood: it takes no seed, top_k, top_p or ras")
    if isinstance(num_samples, bool) or not isinstance(num_samples, (int, np.integer)) or num_samples != 1:
        raise ValueError("num_beams > 1 cannot be combined with num_samples")
    if sample_on_host:
        raise ValueError("num_beams > 1 searches on the device; it cannot be combined with sample_on_host = True")
    if trace is not None or forced is not None:
        raise ValueError("num_beams > 1 cannot be combined with the trace / forced test hooks")
    if fp8:
        raise ValueError("num_beams > 1 is not supported on the FP8 KV cache")
    return n


def _candidates(B: int, n: int, seed, per_utt: Dict[str, object], ras):
    """The arguments of the repeated list that candidate j of utterance b stands for, row b * n + j: every
    per-utterance sequence (checked to hold B values) repeated n times, and the seeds s + b * n + j for an int s, or
    seed[b] + j for B seeds"""
    def rep(v, what):
        v = list(v)
        if len(v) != B:
            raise ValueError(f"{what}: {len(v)} values for {B} utterances")
        return [x for x in v for _ in range(n)]
    if _is_seq(seed):
        if len(seed) != B:
            raise ValueError(f"seed: {len(seed)} values for {B} utterances")
        seeds = [int(s) + j for s in seed for j in range(n)]
    else:
        seeds = int(seed)        # s + r for row r = b * n + j, as the repeated list draws
    out = {k: rep(v, k) if _is_seq(v) else v for k, v in per_utt.items()}
    if _is_seq(ras) and len(ras) > 0 and (ras[0] is None or _is_seq(ras[0])):
        ras = rep(ras, "ras")
    return seeds, out, ras


def _seg_ranges(starts, lens):
    """Concatenated aranges: rows = [starts[b] + i for b for i in range(lens[b])], pos = the i's (int64 numpy)."""
    starts = np.asarray(starts, dtype=np.int64)
    lens = np.asarray(lens, dtype=np.int64)
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    seg_first = np.repeat(np.cumsum(lens) - lens, lens)
    pos = np.arange(total, dtype=np.int64) - seg_first
    return np.repeat(starts, lens) + pos, pos


class ValleEngine:
    """Batched VALLE.inference / VALLE.continual (valle.py:961-1238) for B independent utterances: prefill of the
    AR decoder with a KV cache, the AR sampling loop as one CUDA-graph replay per token with the stop rule on the
    device (valle.py:1012-1057), then the 7 NAR passes (valle.py:1059-1137) over packed ragged rows.  Per utterance the
    result is exactly what the reference's batch-1 call returns; everything below this class is the C ABI."""
    def __init__(self, model, dtype: torch.dtype = torch.float32, use_cuda_graph: bool = True):
        self.lib = L.load()
        self.model = model
        self.dtype = dtype
        self.use_cuda_graph = use_cuda_graph
        p = model.ar_predict_layer.weight
        if not p.is_cuda:
            raise L.VbError("valle_b200: move the model to a CUDA device first (no CPU fallback)")
        self.device = p.device
        self.d = p.shape[1]
        #: width of the NAR stack (valle.py:83: nar_d_model = d_model * nar_scale_factor)
        self.d_nar = model.nar_audio_embeddings[0].weight.shape[1] if model.num_quantizers > 1 else self.d
        #: AR sequences start with <BOS> (id 1025) ahead of the acoustic prompt (valle.py:1006-1007)
        self.prepend_bos = bool(getattr(model, "ar_audio_prepend_bos", False))
        self.n_vocab = p.shape[0]
        self.Q = model.num_quantizers
        self.prefix_mode = model.prefix_mode
        self.stats = EngineStats()
        self.quiet = False
        #: top_k != 1 only: draw on the host exactly as the reference does (logits -> CPU, torch's CPU generator,
        #: one utterance after the other), so that a fixed torch.manual_seed reproduces the reference's ids; the
        #: default draws on the device (torch.multinomial on CUDA logits, Philox stream) without a per-token sync
        self.sample_on_host = False
        self.last_packed: Optional[torch.Tensor] = None
        #: rows of one tensor-core decode group (gemm_decode.cu: one UMMA N tile); larger bf16 batches are split
        self.max_tc_batch = 64
        #: decode steps that draw on the device (greedy or seeded) captured per CUDA graph (one replay per group; the stop
        #: flags are polled every `poll` steps)
        self.steps_per_graph = 8
        self.replayed_launches = 0   # kernels executed through CUDA-graph replays
        self.captured_launches = 0   # kernels recorded at capture time (counted by the library, not run)
        self._bufs: Dict[Tuple[int, int, int], _ArBuffers] = {}
        self._ada_cache = None
        self._sig = None
        self._refresh()

    # ---- weights -----------------------------------------------------------------------
    def _signature(self):
        return tuple((q.data_ptr(), q._version) for q in list(self.model.parameters()) + list(self.model.buffers()))

    def _refresh(self):
        sig = self._signature()
        if sig == self._sig:
            return
        m = self.model
        self._sig = sig
        self.ar = m.ar_decoder.native(self.dtype)
        self.nar = m.nar_decoder.native(self.dtype) if self.Q > 1 else None
        cast = (lambda t: t.detach().to(self.dtype).contiguous()) if self.dtype != torch.float32 \
            else (lambda t: t.detach())
        self.ar_predict_w = cast(m.ar_predict_layer.weight)
        # bf16 pre-LN decode steps run the LayerNorm-folded chain (6 launches per layer instead of 8): the LayerNorms
        # folded into the projections that consume them (vb_ln_fold), incl. the final norm into ar_predict_layer
        # (valle.py:1039).  VB_DECODE_FOLD=0 keeps the 8-launch chain, which post-LN stacks always run.
        self.ar_head_fold = None
        fn = m.ar_decoder.norm
        fold = os.environ.get("VB_DECODE_FOLD", "1") != "0"
        if self.dtype == torch.bfloat16 and fold and fn is not None and self.ar.enable_decode_fold():
            self.ar_head_fold = self.ar.fold_layernorm(self.ar_predict_w, fn.weight.detach(), fn.bias.detach(), None)
        self.nar_predict_w = [cast(l.weight) for l in m.nar_predict_layers] if self.Q > 1 else []
        self._ada_cache = None
        self._bufs.clear()  # graphs hold stale weight pointers
        self._prep_prenets()

    # ---- pre-nets (add_prenet=True, valle.py:96-131,181-214; eval mode: Dropout = identity, BatchNorm1d on its
    #      running statistics) ------------------------------------------------------------------
    def _prep_prenets(self):
        """fp32 weights of the four pre-nets in the layout the kernels take: every Conv1d(k=5, 'same') + BatchNorm1d
        pair becomes ONE [Cout, 5 Cin] matrix (the batch-norm scale / shift folded into weight and bias, columns in
        shift-major order to match `_im2col`), and the AR audio pre-net -- a function of the single embedded token
        (valle.py:1013-1014) -- becomes a pre-computed table over the 1025 (+BOS) ids."""
        m = self.model
        self.pre = None
        self.ar_audio_table = m.ar_audio_embedding.weight.detach()
        if not getattr(m, "add_prenet", False):
            return

        def text(seq):
            convs = []
            for i in (1, 5, 9):
                conv, bn = seq[i], seq[i + 1]
                scale = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).detach().float()
                w = conv.weight.detach().float() * scale[:, None, None]                   # [Cout, Cin, 5]
                b = (conv.bias.detach().float() - bn.running_mean.float()) * scale + bn.bias.detach().float()
                convs.append((w.permute(0, 2, 1).reshape(w.shape[0], -1).contiguous(), b.contiguous()))
            return convs, (seq[14].weight.detach().float().contiguous(), seq[14].bias.detach().float().contiguous())

        def audio(seq):
            return [(seq[i].weight.detach().float().contiguous(), seq[i].bias.detach().float().contiguous())
                    for i in (0, 3, 6)]

        self.pre = {"ar_text": text(m.ar_text_prenet), "ar_audio": audio(m.ar_audio_prenet)}
        if self.Q > 1:
            self.pre["nar_text"] = text(m.nar_text_prenet)
            self.pre["nar_audio"] = audio(m.nar_audio_prenet)
        self.ar_audio_table = self._audio_prenet(m.ar_audio_embedding.weight.detach().float().contiguous(), "ar_audio")

    def _audio_prenet(self, x: torch.Tensor, which: str) -> torch.Tensor:
        (w1, b1), (w2, b2), (w3, b3) = self.pre[which]
        h = ops.linear(x, w1, b1, L.VB_EPI_RELU)
        h = ops.linear(h, w2, b2, L.VB_EPI_RELU)
        return ops.linear(h, w3, b3, L.VB_EPI_NONE)

    def _text_prenet(self, x: torch.Tensor, S: Sequence[int], which: str) -> torch.Tensor:
        """x: packed [sum(S), d] embedded phonemes, utterance after utterance -> the pre-net output, same layout; every
        utterance is convolved on its own with zero padding, as the reference's batch-1 call does (valle.py:995-996)"""
        convs, (wl, bl) = self.pre[which]
        R, d = x.shape
        base, pos = _seg_ranges(_offsets(S)[:-1], S)         # row index, position inside its utterance
        lens = np.repeat(np.asarray(S, dtype=np.int64), S)
        idx = np.stack([np.where((pos + k - 2 >= 0) & (pos + k - 2 < lens), base + k - 2, -1) for k in range(5)])
        idx_d = torch.from_numpy(idx.astype(np.int32)).to(self.device)
        for (w, b) in convs:
            xc = torch.empty((R, 5 * d), dtype=torch.float32, device=self.device)
            for k in range(5):
                ops.gather_rows(x, idx_d[k], out=xc[:, k * d:(k + 1) * d])
            x = ops.linear(xc, w, b, L.VB_EPI_RELU)
        return ops.linear(x, wl, bl, L.VB_EPI_NONE)

    def _pe(self, module, n: int) -> torch.Tensor:
        return module.table(n, self.device)

    def _ada_tables(self) -> List[torch.Tensor]:
        if self._ada_cache is None:
            self._ada_cache = [self.nar.ada_table(e.weight) for e in self.model.nar_stage_embeddings]
        return self._ada_cache

    def _head(self, pe: torch.Tensor, greedy: int) -> L.ArHead:
        m = self.model
        h = L.ArHead()
        h.predict_w = self.ar_predict_w.data_ptr()
        h.n_vocab, h.eos_id = self.n_vocab, NUM_AUDIO_TOKENS
        h.audio_emb = self.ar_audio_table.data_ptr()      # the embedding table, or pre-net(embedding) (add_prenet)
        h.alpha = m.ar_audio_position.alpha.detach().data_ptr()
        h.pe, h.pe_rows = pe.data_ptr(), pe.shape[0]
        h.greedy = int(greedy)
        if self.ar_head_fold is not None:
            h.fold = self.ar_head_fold
        return h

    def kv_cache_dtype(self) -> Optional[torch.dtype]:
        """the model's `kv_cache_dtype` (None: the cache holds the engine dtype), validated against the engine dtype"""
        kv = getattr(self.model, "kv_cache_dtype", None)
        if kv is None:
            return None
        if kv != torch.float8_e4m3fn:
            raise ValueError(f"kv_cache_dtype={kv}: only None (the engine dtype) and torch.float8_e4m3fn are supported")
        if self.dtype != torch.bfloat16:
            raise ValueError(f"kv_cache_dtype=torch.float8_e4m3fn needs engine_dtype=torch.bfloat16 (got {self.dtype})")
        return kv

    def _buffers(self, B: int, cap: int, tok_stride: int, kv_dtype: Optional[torch.dtype] = None) -> _ArBuffers:
        key = (B, cap, tok_stride, kv_dtype)
        b = self._bufs.get(key)
        if b is None:
            if len(self._bufs) > 4:
                self._bufs.clear()
            b = _ArBuffers(self, B, cap, tok_stride, kv_dtype)
            self._bufs[key] = b
        return b

    # ---- public API ----------------------------------------------------------------------
    @torch.no_grad()
    @_on_device
    def generate(self, texts: Sequence[torch.Tensor], prompts: Sequence[torch.Tensor],
                 enroll_lens: Optional[Sequence[int]] = None, top_k: int = 1, temperature: float = 1.0,
                 max_new_tokens=None, poll: int = 32,
                 return_device: bool = False, trace: Optional[dict] = None,
                 forced: Optional[Sequence[torch.Tensor]] = None, seed=None, top_p=1.0,
                 ras=None, num_samples: int = 1, return_scores: bool = False, num_beams: int = 1):
        """texts[b]: int64 [S_b] phoneme ids; prompts[b]: int64 [Tp_b, Q] codec ids (host or device).
        Returns codes[b]: int64 [Tgen_b, Q] -- per utterance exactly what VALLE.inference returns.

        seed: None draws top_k != 1 ids with torch's generator (torch.multinomial on the device, or on the host with
        `sample_on_host`).  An int s, or a sequence of B ints in [0, 2**64), selects the seeded device sampler
        (vb_sample_logits): utterance b draws from seed s + b (or seed[b]) and its decode step, inside the CUDA-graph
        decode step, so its codes do not depend on the batch it shares, its slot, or how the call is split.  With a
        seed, top_k, temperature and top_p may be per-utterance sequences; every top_k == 1 without ras is the greedy
        path.  max_new_tokens: None, one int, or a sequence of B ints (one cap per utterance).
        top_p: nucleus filtering after top-k (valle.py:1242-1284), in (0, 1]; 1 is off.  Without a seed it goes to the
        reference's own topk_sampling.
        ras: repetition-aware sampling (VALL-E 2), seeded calls only: a (window, threshold) pair, or one pair / None per
        utterance.  A draw that already makes up more than `threshold` of the utterance's last `window` codes (window
        in [1, 256], threshold in [0, 1)) is replaced by a draw from the unfiltered distribution; see
        include/valle_b200.h vb_sample_logits_ex.

        Best-of-n (seeded calls only): num_samples=n > 1 draws n candidates per utterance and returns codes[b][j], B
        lists of n [T, Q] tensors.  Candidate j of utterance b draws from seed s + b * n + j (int s) or seed[b] + j (B
        seeds), and its codes are bit for bit those of generate() on the list with every utterance repeated n times;
        on the bf16 and fp32 caches the n candidates' decode steps read one copy of their shared prompt prefix from the
        KV cache.  One caveat, the batch-size caveat every batched call carries: in bf16 a decode group holds
        floor(64 / n) whole utterances, so with B * n > 64 and n not dividing 64 the groups differ from the repeated
        list's groups of 64 rows, and the default KV split count (which depends on the group's size) may then round a
        row's attention differently.  With VB_DECODE_NSPLIT fixed the codes are the repeated list's in every case.
        return_scores=True (any seeded call) returns (codes, scores): scores [B, n] fp32, the AR log-likelihood of each
        candidate, the sum over its first-codebook codes of log_softmax(raw logits)[code] (before temperature, top-k
        and top-p), accumulated in fp32 on the device.

        Beam search: num_beams=n > 1 (an int in [1, 16]; no seed, top_k, top_p, ras, num_samples, host sampling, test
        hooks or FP8 KV cache) keeps the n most likely first-codebook hypotheses of each utterance and returns one [T, Q]
        code matrix per utterance, its first codebook the winning hypothesis, the NAR run once on it; include/
        valle_b200.h "Beam search" states the ranking and the exact stop rule (no length normalisation).
        return_scores=True returns (codes, scores [B] fp32), the winner's AR log-likelihood over its codes.  The n
        beams of an utterance are n decode rows that read one copy of the prompt prefix, and the batch caveat of
        best-of-n applies: in bf16 a decode group holds floor(64 / n) whole utterances; with VB_DECODE_NSPLIT fixed an
        utterance's result does not depend on its batch.  num_beams=1 runs the default path.

        Test hooks: `trace` collects AR logits (trace["steps"] = set of iterations or "all") and, with
        trace["nar"] = True, the NAR logits / argmax of every stage; `forced[b]` = int64 [T_b, Q] codes the decode is
        teacher-forced with (every sampled id is replaced by the given one before it is appended, AR and NAR), so
        that per-step logits can be compared with a reference that took exactly those ids."""
        self._refresh()
        B = len(texts)
        if B < 1 or len(prompts) != B:
            raise ValueError(f"generate: {B} texts and {len(prompts)} prompts (one of each per utterance, >= 1)")
        bf16 = self.dtype == torch.bfloat16
        beams = _check_num_beams(num_beams, seed, top_k, top_p, ras, num_samples, trace, forced, self.sample_on_host,
                                 self.kv_cache_dtype() is not None) > 1
        if beams:
            n = int(num_beams)
        else:
            n = _check_num_samples(num_samples, seed, return_scores, trace, forced, self.sample_on_host,
                                   self.max_tc_batch if bf16 else None)
        if n > 1:
            seeds, per, ras = _candidates(B, n, 0 if beams else seed,
                                          dict(texts=texts, prompts=prompts, enroll_lens=enroll_lens,
                                               max_new_tokens=max_new_tokens, top_k=top_k,
                                               temperature=temperature, top_p=top_p), ras)
            seed = None if beams else seeds
            texts, prompts, enroll_lens, max_new_tokens = (per[k] for k in ("texts", "prompts", "enroll_lens",
                                                                            "max_new_tokens"))
            top_k, temperature, top_p = per["top_k"], per["temperature"], per["top_p"]
        rows = B * n
        draws = None
        if ras is not None and self.sample_on_host:
            raise ValueError("ras draws on the device; it cannot be combined with sample_on_host = True")
        if seed is not None:
            if self.sample_on_host:
                raise ValueError("seed= selects the device sampler; it cannot be combined with sample_on_host = True")
            draws = _draws(rows, seed, top_k, temperature, top_p, ras)
            if all(dr.greedy for dr in draws) and not return_scores:
                draws, top_k = None, 1          # greedy: the seed draws nothing (scores keep the seeded sampler)
        elif ras is not None:
            raise ValueError("ras needs seed= (the seeded device sampler)")
        elif _is_seq(top_k) or _is_seq(temperature) or _is_seq(top_p):
            raise ValueError("per-utterance top_k / temperature / top_p need seed= (the seeded device sampler)")
        else:
            top_p = float(top_p)
            _check_top_p([top_p])
        if not (rows > self.max_tc_batch and bf16 and trace is None and forced is None):
            outs, scores = self._generate(texts, prompts, enroll_lens, draws, top_k, temperature, top_p,
                                          max_new_tokens, poll, return_device, trace, forced, n, return_scores, beams)
            return self._best_of(outs, scores, B, n, return_scores, return_device, beams)
        # the tensor-core decode projections take up to 64 rows (one UMMA N tile): a larger batch is decoded as
        # consecutive groups of <= 64 rows instead of falling onto the CUDA-core GEMV path; a group holds whole
        # utterances, all n candidates of each
        group = self.max_tc_batch // n * n
        outs: List[torch.Tensor] = []
        scores = []
        stats = EngineStats()
        packed = []
        for b0 in range(0, rows, group):
            b1 = min(rows, b0 + group)
            mnt = max_new_tokens[b0:b1] if _is_seq(max_new_tokens) else max_new_tokens
            o, sc = self._generate(texts[b0:b1], prompts[b0:b1], None if enroll_lens is None else enroll_lens[b0:b1],
                                   None if draws is None else draws[b0:b1], top_k, temperature, top_p, mnt, poll,
                                   return_device, num_samples=n, scores=return_scores, beams=beams)
            outs += o
            scores.append(sc)
            stats.ar_steps += self.stats.ar_steps
            stats.ar_ms += self.stats.ar_ms
            stats.prefill_ms += self.stats.prefill_ms
            stats.nar_ms += self.stats.nar_ms
            packed.append(self.last_packed)
        self.stats = stats
        self.last_packed = torch.cat(packed) if return_device else None
        return self._best_of(outs, torch.cat(scores) if return_scores else None, B, n, return_scores, return_device,
                             beams)

    @staticmethod
    def _best_of(outs: List[torch.Tensor], scores: Optional[torch.Tensor], B: int, n: int, return_scores: bool,
                 return_device: bool, beams: bool = False):
        """generate()'s result from the codes of its B * n rows and their scores: the rows grouped per utterance when
        n > 1, and (codes, scores [B, n]) with return_scores.  beams: outs and scores hold one entry per utterance
        already (scores [B])."""
        codes = outs if n == 1 or beams else [outs[b * n:(b + 1) * n] for b in range(B)]
        if not return_scores:
            return codes
        scores = scores.view(B) if beams else scores.view(B, n)
        return codes, scores if return_device else scores.cpu()

    def _generate(self, texts, prompts, enroll_lens, draws: Optional[List[_Draw]], top_k, temperature, top_p,
                  max_new_tokens, poll: int, return_device: bool, trace: Optional[dict] = None,
                  forced: Optional[Sequence[torch.Tensor]] = None, num_samples: int = 1,
                  scores: bool = False, beams: bool = False) -> Tuple[List[torch.Tensor], Optional[torch.Tensor]]:
        """generate() of one group of utterances with validated sampler arguments: draws (the seeded device sampler), or
        None and top_k / temperature / top_p (greedy, or torch's sampler).  num_samples > 1: the rows are the
        candidates of B / num_samples utterances, num_samples consecutive rows each, which decode reading their first row's prompt prefix.  Returns the
        codes and, with scores (seeded draws only), the rows' AR log-likelihoods on the device.  beams: the rows are
        the beams of B / num_samples utterances (beam search); returns one code matrix and score per utterance."""
        m, dev, Q = self.model, self.device, self.Q
        B = len(texts)
        kv_dtype = self.kv_cache_dtype()
        for b in range(B):
            _check_utt(f"utterance {b}", texts[b], prompts[b], Q)
        if self.prefix_mode in (2, 4) and Q > 1 and enroll_lens is None:
            raise ValueError(f"prefix_mode {self.prefix_mode} needs enroll_lens (the NAR text leaves them out)")
        S = [int(t.numel()) for t in texts]
        Tp = [int(p.shape[0]) for p in prompts]
        cap_new = self._cap_new(S, max_new_tokens)
        tok_stride = (max(cap_new) + 2 + 7) // 8 * 8
        cap = (max(S[b] + Tp[b] + cap_new[b] + 2 for b in range(B)) + 63) // 64 * 64
        greedy = draws is None and top_k == 1 and forced is None
        # seeded draw in the decode step's tail (forced ids replace every draw: that runs the push path below)
        native = draws is not None and forced is None
        forced_steps = None
        if forced is not None:  # [steps, B] first-codebook ids, EOS once an utterance's forced ids run out
            n_f = max(int(f.shape[0]) for f in forced) + 1
            forced_steps = torch.full((n_f + 1, B), NUM_AUDIO_TOKENS, dtype=torch.int64)
            for b, f in enumerate(forced):
                forced_steps[: f.shape[0], b] = f[:, 0].to(torch.int64).cpu()
            forced_steps = forced_steps.to(dev)
            cap_new = [min(c, int(f.shape[0])) for c, f in zip(cap_new, forced)]

        # ---- host -> device (once per batch) ----
        p = self._prefill_inputs(texts, prompts, cap_new)
        utts = p.utts(range(B), [None] * B if enroll_lens is None else enroll_lens)

        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        # ---- AR prefill (valle.py:995-997,1013-1016) ----
        buf = self._buffers(B, cap, tok_stride, kv_dtype)
        buf.load_rows(p, draws if native else None)
        buf.n_gen.zero_()
        buf.finished.zero_()
        buf.set_best_of(B, num_samples, scores and not beams, beams)
        pe_a = self._pe(m.ar_audio_position, max(p.Tp) + max(cap_new) + 2)
        h_last = self._prefill(buf, p, pe_a)
        head = self._head(pe_a, 3 if beams else 2 if native else int(greedy))
        self._head_ref = head
        L.check(self.lib.vb_ar_head_step(self.ar.handle, C.byref(head), h_last.data_ptr(), C.byref(buf.st),
                                         buf.ws.data_ptr(), buf.ws.numel(), L.stream_ptr()), "vb_ar_head_step")
        def want(step):
            st_ = trace.get("steps", ())
            return st_ == "all" or step in st_
        if trace is not None:  # test hook: AR logits of selected iterations (iteration 0 = prefill)
            trace.setdefault("ar_logits", {})
            if want(0):
                trace["ar_logits"][0] = buf.logits[:, : self.n_vocab].clone()
            poll = 1
        if forced_steps is not None:
            poll = 1
        if not (greedy or native):
            self._sample_push(buf, head, top_k, temperature, None if forced_steps is None else forced_steps[0], top_p)
        if any(t.is_cuda for t in list(texts) + list(prompts)):
            ops.check_oob(dev)  # ids that were already on the device are range-checked by the embedding kernels
        ev[1].record()

        # ---- AR decode loop (valle.py:1012-1057) ----
        max_steps = max(cap_new) + 1     # the stop rule has fired in every row by then
        steps = 0
        # beam search: the first row of each group stands for its utterance (it receives the result)
        rows = list(range(0, B, num_samples)) if beams else list(range(B))
        utts = [utts[r] for r in rows]
        running = dict(zip(rows, utts))
        Tg_row = {}
        while running and steps < max_steps:
            n = min(poll, max_steps - steps)
            if (greedy or native) and self.use_cuda_graph:
                self._device_steps(buf, head, n)
            else:
                for _ in range(n):
                    self._launch_step(buf, head)
                    if not (greedy or native):   # draw on the host, or take the forced ids
                        fs = None
                        if forced_steps is not None:
                            fs = forced_steps[min(steps + 1, forced_steps.shape[0] - 1)]
                        self._sample_push(buf, head, top_k, temperature, fs, top_p)
            steps += n
            if trace is not None and want(steps):  # poll == 1 here: the logits row of iteration `steps`
                trace["ar_logits"][steps] = buf.logits[:, : self.n_vocab].clone()
            for b, n_b in self._stopped(buf, running).items():
                Tg_row[b] = n_b
                del running[b]
        Tg = [Tg_row.get(r, 0) for r in rows]
        self.stats.ar_steps = steps
        if beams:
            logprob = buf.beam_score[rows].clone() if scores else None
        else:
            logprob = buf.logprob[:B].clone() if scores else None
        ev[2].record()

        # ---- NAR (valle.py:1059-1137) ----
        src = torch.from_numpy(_seg_ranges(np.asarray(rows, dtype=np.int64) * tok_stride, Tg)[0]).to(dev)
        fc = None
        if forced is not None:
            fc = torch.cat([forced[b][: Tg[b]].to(torch.int64) for b in range(B)]).to(dev)
        codes, cu_g = self._nar(utts, Tg, buf.tokens.view(-1).index_select(0, src).to(torch.int64), forced_codes=fc,
                                trace=trace if (trace is not None and trace.get("nar")) else None)
        ev[3].record()
        ev[3].synchronize()
        if any(t.is_cuda for t in list(texts) + list(prompts)):
            ops.check_oob(dev)
        self.stats.prefill_ms = ev[0].elapsed_time(ev[1])
        self.stats.ar_ms = ev[1].elapsed_time(ev[2])
        self.stats.nar_ms = ev[2].elapsed_time(ev[3])
        #: the packed [sum(Tgen), Q] device tensor behind the returned per-utterance views (dist.gather_codes ships it
        #: as is instead of re-packing the views)
        self.last_packed = codes
        if return_device:
            return [codes[cu_g[b]:cu_g[b + 1]] for b in range(len(rows))], logprob
        host = codes.cpu()
        return [host[cu_g[b]:cu_g[b + 1]] for b in range(len(rows))], logprob

    def generate_stream(self, requests: Iterable, slots: Optional[int] = None, max_context: Optional[int] = None,
                        poll: int = 32, nar_batch: Optional[int] = None, return_scores: bool = False) -> Iterator[tuple]:
        """Continuous batching: decode `requests` (StreamRequest or BestOfRequest records, or tuples in
        StreamRequest's field order) in `slots`
        decode rows, refilling a row with the next request as soon as its utterance stops, and yield (index, codes) in
        completion order.  codes: int64 [Tgen, Q] on the device, what generate() returns for that utterance; index:
        the request's position in `requests`.

        requests may be a lazy iterator (pulled from while decoding runs); the KV cache holds `max_context` rows per
        slot (text + prompt + new tokens + 2; default: the largest request of a sequence, required for an iterator),
        and a request that needs more raises ValueError when it is pulled.  slots: default min(#requests, 64); bf16
        takes at most 64 (one tensor-core decode group).  New requests are admitted, and the stop flags read, every
        `poll` decode steps; the NAR runs over every `nar_batch` (default `slots`) finished utterances, and over the
        rest once nothing is left to decode.  Sampling is greedy, or seeded per request (`seed`, with top_k /
        temperature / top_p / ras): the draws depend on the seed, the step and the request's own codes only, never on
        the slot or the schedule.  A request with num_beams=n > 1 is decoded by beam search (generate(num_beams=n)'s
        rules; not on the FP8 cache, n <= slots) in n consecutive slots that read one copy of its prompt prefix and are
        freed together; requests are admitted first in, first out, so one that finds no run of n free slots waits, and
        the requests behind it with it.  Its codes are those of generate(num_beams=n) on it alone.

        A BestOfRequest(request, n) (a seed s, n <= slots, no beams) decodes n seeded candidates in n consecutive
        slots, candidate j drawing from seed s + j, and yields the list of their n codes, bit for bit
        generate([text], [prompt], seed=s, num_samples=n)[0] (with the KV split count caveat of any batch).  On the
        bf16 and fp32 caches the request is prefilled once, into its first slot, whose prompt prefix the other
        candidates read; that slot is held until every candidate has stopped, every other one is freed as its
        candidate stops.  On the FP8 cache each candidate is a row of its own.  The candidates go to the NAR as they
        stop (nar_batch counts candidates); the request is yielded once all n are through.

        return_scores=True yields (index, codes, scores): scores a device fp32 tensor, what
        generate(..., return_scores=True, return_device=True)[1][0] gives for the request alone: [1] for a request,
        [n] for a best-of request, the winner's score (0-d) for a beam request.  A greedy request without a seed is
        scored as generate(seed=0) scores it; every request then runs the seeded sampler's head."""
        with torch.cuda.device(self.device):
            self._refresh()
        kv_dtype = self.kv_cache_dtype()
        if self.sample_on_host:
            raise ValueError("generate_stream draws on the device: sample_on_host = True is not supported")
        if isinstance(requests, (list, tuple)):
            reqs = [_as_request(r) for r in requests]
            if not reqs:
                return iter(())
            if max_context is None:
                max_context = max(self._context(r.request if isinstance(r, BestOfRequest) else r) for r in reqs)

            def rows(r):   # the candidates of a best-of request (validated when the request is pulled)
                n = r.num_samples if isinstance(r, BestOfRequest) else 1
                return int(n) if isinstance(n, (int, np.integer)) and not isinstance(n, bool) and n > 1 else 1
            slots = min(sum(rows(r) for r in reqs), self.max_tc_batch) if slots is None else slots
            it = iter(reqs)
        else:
            if max_context is None:
                raise ValueError("generate_stream: an iterator of requests needs max_context")
            slots = self.max_tc_batch if slots is None else slots
            it = (_as_request(r) for r in requests)
        slots, poll = int(slots), int(poll)
        nar_batch = slots if nar_batch is None else int(nar_batch)
        if slots < 1 or poll < 1 or nar_batch < 1:
            raise ValueError("generate_stream: slots, poll and nar_batch must be >= 1")
        if self.dtype == torch.bfloat16 and slots > self.max_tc_batch:
            raise ValueError(f"generate_stream: bf16 decodes at most {self.max_tc_batch} slots (got {slots})")
        return self._stream(it, slots, int(max_context), poll, nar_batch, kv_dtype, bool(return_scores))

    def _context(self, r: StreamRequest) -> int:
        """KV-cache rows a request needs: text + prompt + the most tokens it may generate + 2"""
        S = int(r.text.numel())
        return S + int(r.prompt.shape[0]) + self._cap_new([S], r.max_new_tokens)[0] + 2

    @torch.no_grad()
    def _stream(self, it, n_slots: int, max_context: int, poll: int, nar_batch: int, kv_dtype, scores: bool = False):
        m, dev, Q = self.model, self.device, self.Q
        cap = (max_context + 63) // 64 * 64
        tok_stride = (max_context + 2 + 7) // 8 * 8
        pm = self.prefix_mode
        # a best-of request's candidates read one prefill of its prompt (kv_parent); the FP8 cache refuses kv_parent,
        # and its shared read is no faster there (DESIGN section 7): each candidate is prefilled into its own slot
        fork = kv_dtype is None
        stats = EngineStats()
        phases: Dict[str, list] = {"prefill_ms": [], "ar_ms": [], "nar_ms": []}

        def timed(name):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            phases[name].append([e])
            return phases[name][-1]

        with torch.cuda.device(dev):
            buf = self._buffers(n_slots, cap, tok_stride, kv_dtype)
            buf.n_gen.zero_()
            buf.finished.fill_(1)              # a slot that is never filled never runs, nor reads its sampler columns
            buf.x_cur.zero_()
            # no shared prefixes yet; logprob zeroed with scores
            buf.set_best_of(n_slots, 1, scores)
            pe_a = self._pe(m.ar_audio_position, cap + 2)
            heads = {g: self._head(pe_a, g) for g in (1, 2, 4)}
            ws = torch.empty(self.lib.vb_ar_admit_workspace(C.byref(self.ar.desc), n_slots, self.n_vocab),
                             dtype=torch.uint8, device=dev)
        # 2 (the seeded sampler) from the first seeded request on, or from the start with scores (scores keep the seeded
        # sampler, as in generate()); 4 (2 next to beam groups) from the first beam request
        mode = 2 if scores else 1
        shared = False                         # a best-of request reads its parent's prompt prefix (kv_parent)
        free = list(range(n_slots))
        # pulled requests waiting for slots, in order: (index, request, the draws of its candidates)
        queue: List[Tuple[int, StreamRequest, List[_Draw]]] = []
        active: Dict[int, _Utt] = {}           # slot -> the utterance decoding in it (a beam group's first slot)
        width: Dict[int, int] = {}             # active slot -> the slots its utterance holds from there on
        cand: Dict[int, Tuple[_Candidates, int]] = {}   # active slot -> its request's candidates, and which one
        # stopped candidates waiting for the NAR: utterance, codes, request, candidate, score
        pending: List[Tuple[_Utt, torch.Tensor, _Candidates, int, Optional[torch.Tensor]]] = []
        n_pulled, exhausted, device_ids = 0, False, False

        def slots_of(q):
            _, r, draws = q
            return r.num_beams if r.num_beams > 1 else len(draws)

        def pull(k):
            """up to k validated requests: (index, request, the draws of its candidates)"""
            nonlocal n_pulled, exhausted, mode, shared
            out = []
            while len(out) < k and not exhausted:
                try:
                    r = next(it)
                except StopIteration:
                    exhausted = True
                    break
                idx = n_pulled
                n_pulled += 1
                r, draws = _stream_draws(idx, r, Q, n_slots, kv_dtype is not None)
                beams = r.num_beams
                if pm in (2, 4) and r.enroll_len is None:
                    raise ValueError(f"request {idx}: prefix_mode {pm} needs enroll_len")
                if self._context(r) > max_context:
                    raise ValueError(f"request {idx} needs {self._context(r)} KV-cache rows > max_context={max_context}")
                if beams > 1:
                    mode = 4
                elif not all(d.greedy for d in draws):
                    mode = max(mode, 2)
                shared |= len(draws) > 1 and fork
                out.append((idx, r, draws))
            return out

        def admit(new, taken):
            """the requests `new`, each into its slots of `taken`: a beam group's n rows are its request n times, the
            prefill writing each row's own cache streams; a best-of request's candidates are its request n times too,
            except where they share its prompt prefix: then its first slot (the parent) is prefilled alone, and the
            other candidates read the prefix below P from it and get the rows from P on copied (vb_ar_fork_prefix)"""
            nonlocal device_ids
            pre, forked = [], []   # (request, slot, candidate, its slots' first, the prefill row it takes)
            for q, ss in zip(new, taken):
                _, r, draws = q
                parent = len(pre)
                for j, sl in enumerate(ss):
                    row = (q, sl, j, ss[0], parent)
                    if j > 0 and len(draws) > 1 and fork:
                        forked.append(row)
                    else:
                        pre.append(row[:4] + (len(pre),))
            rows = pre + forked
            texts = [q[1].text for q, *_ in pre]
            prompts = [q[1].prompt for q, *_ in pre]
            cap_new = [self._cap_new([int(q[1].text.numel())], q[1].max_new_tokens)[0] for q, *_ in pre]
            p = self._prefill_inputs(texts, prompts, cap_new, slots=[sl for _, sl, *_ in pre],
                                     forks=([sl for _, sl, *_ in forked], [i for *_, i in forked]) if forked else None)
            ev = timed("prefill_ms")
            # each row's kv_parent: a beam group's and a shared best-of request's first slot, else the row itself
            kvp = [first if q[1].num_beams > 1 or (len(q[2]) > 1 and fork) else sl for q, sl, _, first, _ in rows]
            groups = parents = None
            if mode == 4:   # (kv_parent, beam_first, beam_n) of each row
                groups = [(kp, first if q[1].num_beams > 1 else -1, slots_of(q))
                          for kp, (q, _, _, first, _) in zip(kvp, rows)]
            elif buf.st.kv_parent is not None:
                parents = kvp
            buf.load_rows(p, [q[2][j if len(q[2]) > 1 else 0] for q, _, j, *_ in rows], groups, parents)
            h = self._prefill(buf, p, pe_a)
            slots_d = p.slots_d
            if forked:
                slots_d = p.admit_d
                h = ops.gather_rows(h, p.gather_d)
                L.check(self.lib.vb_ar_fork_prefix(self.ar.handle, p.admit_d[len(pre):].data_ptr(), len(forked),
                                                   C.byref(buf.st), L.stream_ptr()), "vb_ar_fork_prefix")
            L.check(self.lib.vb_ar_admit(self.ar.handle, C.byref(heads[mode]), h.data_ptr(), len(rows),
                                         slots_d.data_ptr(), C.byref(buf.st), ws.data_ptr(), ws.numel(),
                                         L.stream_ptr()), "vb_ar_admit")
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev.append(e)
            utts = p.utts([q[0] for q, *_ in pre], [q[1].enroll_len for q, *_ in pre])
            reqs = {}
            for q, ss in zip(new, taken):
                idx, r, draws = q
                beam = r.num_beams > 1
                reqs[idx] = _Candidates(idx, 1 if beam else len(draws), ss[0] if len(draws) > 1 and fork else None,
                                        len(draws) > 1, beam)
            for q, sl, j, first, i in rows:
                if q[1].num_beams > 1 and sl != first:
                    continue   # a beam group decodes as its first slot
                active[sl], width[sl], cand[sl] = utts[i], slots_of(q) if q[1].num_beams > 1 else 1, (reqs[q[0]], j)
                reqs[q[0]].running.add(sl)
            device_ids |= any(t.is_cuda for t in texts + prompts)
            stats.admissions += len(new)

        def nar(batch):
            ev = timed("nar_ms")
            codes, cu_g = self._nar([u for u, *_ in batch], [int(c.shape[0]) for _, c, *_ in batch],
                                    torch.cat([c for _, c, *_ in batch]))
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev.append(e)
            out = []
            for i, (_, _, req, j, sc) in enumerate(batch):
                if req.done(j, codes[cu_g[i]:cu_g[i + 1]], sc):
                    out.append(req.result(scores))
            return out

        def advance():
            """admission, `poll` decode steps and the stop flags; returns the requests whose codes are ready"""
            if free and (queue or not exhausted):
                queue.extend(pull(len(free) - len(queue)))
                if mode == 4 and buf.st.beam_first is None:
                    buf.set_groups(parents=buf.st.kv_parent is None)
                if shared and buf.st.kv_parent is None:
                    buf.set_parents()
                taken = _take_slots(free, [slots_of(q) for q in queue])
                if taken:
                    admit(queue[:len(taken)], taken)
                    del queue[:len(taken)]
            if active:
                ev = timed("ar_ms")
                head = heads[mode]
                if self.use_cuda_graph:
                    self._device_steps(buf, head, poll)
                else:
                    for _ in range(poll):
                        self._launch_step(buf, head)
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                ev.append(e)
                stats.ar_steps += poll
                for s, n in self._stopped(buf, active).items():
                    w = width.pop(s)
                    req, j = cand.pop(s)
                    # copied out now: the slot may be refilled before the NAR batch runs
                    sc = (buf.beam_score if w > 1 else buf.logprob)[s].clone() if scores else None
                    pending.append((active.pop(s), buf.tokens[s, :n].to(torch.int64), req, j, sc))
                    freed = req.stop(s)
                    if w > 1:   # its rows leave the group: any request may take any of them
                        buf.beam_first[s:s + w] = -1
                        freed = list(range(s, s + w))
                    stats.slot_steps += n * w
                    free.extend(freed)
                free.sort()
            ready = []
            drain = exhausted and not active and not queue
            while len(pending) >= nar_batch or (drain and pending):
                batch = pending[:nar_batch]
                del pending[:nar_batch]
                ready += nar(batch)
            if device_ids:
                ops.check_oob(dev)
            return ready

        while True:
            with torch.cuda.device(dev):
                ready = advance()
            yield from ready
            if exhausted and not active and not pending and not queue:
                break
        torch.cuda.synchronize(dev)
        for name, evs in phases.items():
            setattr(stats, name, sum(a.elapsed_time(b) for a, b in evs))
        self.stats = stats

    # ---- shared by generate() and generate_stream() ----------------------------------------
    def _cap_new(self, S: Sequence[int], max_new_tokens) -> List[int]:
        """per utterance: the n_gen past which the stop rule fires (valle.py:1047: n_new > 16 * S), lowered to
        max_new_tokens - 1 (one int, or one per utterance)"""
        cap_new = [16 * s for s in S]
        if self.prepend_bos:
            # y carries the <BOS> the prompt does not: (y.shape[1] - prompts.shape[1]) = n_new + 1 (valle.py:1045-1047)
            cap_new = [c - 1 for c in cap_new]
        if max_new_tokens is not None:
            mnt = [int(x) for x in max_new_tokens] if _is_seq(max_new_tokens) else [int(max_new_tokens)] * len(S)
            if len(mnt) != len(S):
                raise ValueError(f"max_new_tokens: {len(mnt)} values for {len(S)} utterances")
            cap_new = [min(c, t - 1) for c, t in zip(cap_new, mnt)]
        return cap_new

    def _stopped(self, buf: _ArBuffers, rows: Dict[int, _Utt]) -> Dict[int, int]:
        """The stop flags and n_gen of buf in one device -> host copy (one sync): of `rows` (row -> its utterance), the
        ones whose utterance has stopped, in row order, with their n_gen.  Prints their EOS lines (valle.py:1054);
        an utterance that stopped before its first code raises as the reference does (valle.py:1049-1052)."""
        fin, n_gen = torch.stack([buf.finished, buf.n_gen]).cpu().tolist()
        out = {}
        for s in sorted(rows):
            if fin[s] == 0:
                continue
            if fin[s] == 2:
                raise SyntaxError("well trained model shouldn't reach here.")
            if not self.quiet:
                print(f"VALL-E EOS [{rows[s].prompt.shape[0]} -> {rows[s].Tp_ar + n_gen[s]}]")
            out[s] = n_gen[s]
        return out

    def _prefill_inputs(self, texts, prompts, cap_new, slots: Optional[Sequence[int]] = None,
                        forks: Optional[Tuple[Sequence[int], Sequence[int]]] = None) -> _Prefill:
        """the host -> device copies of one packed AR prefill (ids, and one int32 block of lengths and row maps);
        slots: the decode slots the utterances go to (generate_stream); forks: (slots, utterances) of rows admitted
        without a prefill of their own, each taking utterance i's (a best-of request's other candidates)"""
        dev, Q = self.device, self.Q
        B = len(texts)
        S = [int(t.numel()) for t in texts]
        Tp = [int(p.shape[0]) for p in prompts]
        text_all = torch.cat([t.reshape(-1).to(torch.int64) for t in texts]).to(dev, non_blocking=True)
        prm_all = torch.cat([p.to(torch.int64) for p in prompts]).contiguous().to(dev, non_blocking=True)
        Tp_nar, ar_tok = Tp, None
        if self.prepend_bos:   # the AR stack sees [<BOS> | first-codebook prompt]; the NAR stages see the prompt only
            bos = torch.full((1,), NUM_AUDIO_TOKENS + 1, dtype=torch.int64)
            ar_tok = torch.cat([torch.cat([bos, p[:, 0].to(torch.int64).cpu()]) for p in prompts]).to(dev, non_blocking=True)
            Tp = [t + 1 for t in Tp]
        seq_len = [S[b] + Tp[b] for b in range(B)]
        cu_np = _offsets(seq_len)
        text_rows, text_pos = _seg_ranges(cu_np[:-1], S)
        aud_rows, aud_pos = _seg_ranges(cu_np[:-1] + np.asarray(S, dtype=np.int64), Tp)
        fs, fi = ([], []) if forks is None else forks
        meta = torch.from_numpy(np.concatenate([cu_np, S, Tp, cap_new, text_rows, text_pos, aud_rows, aud_pos,
                                                cu_np[1:] - 1, [] if slots is None else slots, fs,
                                                [] if forks is None else list(range(B)) + list(fi)]).astype(np.int32)
                                ).to(dev, non_blocking=True)
        sizes = [B + 1, B, B, B, sum(S), sum(S), sum(Tp), sum(Tp), B, 0 if slots is None else B]
        v = meta.split(sizes + [len(fs), len(fs) + B if forks else 0])
        admit_d = gather_d = None
        if forks is not None:   # slots_d and the forked rows' slots, as one array
            admit_d, gather_d = meta.narrow(0, sum(sizes) - B, B + len(fs)), v[-1]
        return _Prefill(S, Tp, Tp_nar, text_all, prm_all, ar_tok, *v[:9], None if slots is None else v[9], admit_d,
                        gather_d)

    def _prefill(self, buf: _ArBuffers, p: _Prefill, pe_a: torch.Tensor) -> torch.Tensor:
        """embedding (+ pre-net) + positions of every [text | prompt] row and the AR prefill (valle.py:995-997,
        1013-1016), which fills cache stream b of buf, or p.slots_d[b]; returns the last row of each utterance [B, d]"""
        m = self.model
        S, Tp = p.S, p.Tp
        pe_t = self._pe(m.ar_text_position, max(S))
        x = torch.empty((sum(S) + sum(Tp), self.d), dtype=torch.float32, device=self.device)
        self._embed_pe(p.text_all, 1, m.ar_text_embedding.weight, pe_t, m.ar_text_position.alpha, sum(S), x, p.trow_d,
                       p.tpos_d, prenet=("ar_text", S) if self.pre else None)
        if self.prepend_bos:
            self._embed_pe(p.ar_tok, 1, self.ar_audio_table, pe_a, m.ar_audio_position.alpha, sum(Tp), x, p.arow_d, p.apos_d)
        else:
            self._embed_pe(p.prm_all, self.Q, self.ar_audio_table, pe_a, m.ar_audio_position.alpha, sum(Tp), x, p.arow_d,
                           p.apos_d)
        self.ar.forward(x, p.cu_d, len(S), max(s + t for s, t in zip(S, Tp)), L.VB_MASK_VALLE_AR, p.S_d, None,
                        buf.kcache, buf.vcache, buf.cap, k_exp=buf.k_exp, v_exp=buf.v_exp, cache_slots=p.slots_d)
        return ops.gather_rows(x, p.last_d)

    def _device_steps(self, buf: _ArBuffers, head: L.ArHead, n: int):
        """n decode steps that draw on the device: whole groups of `steps_per_graph` steps as one graph replay (no launch
        gap between the steps of a group), the remainder one step at a time"""
        done = 0
        while done < n:
            k = self.steps_per_graph if n - done >= self.steps_per_graph else 1
            self._replay_steps(buf, head, k)
            done += k

    @torch.no_grad()
    @_on_device
    def continual(self, texts: Sequence[torch.Tensor], ys: Sequence[torch.Tensor]) -> List[torch.Tensor]:
        """VALLE.continual (valle.py:1139-1238): first-codebook codes are given, the 7 NAR stages
        predict the rest; prefix = min(T // 2, 225) frames."""
        self._refresh()
        dev, Q = self.device, self.Q
        B = len(texts)
        for b in range(B):
            _check_utt(f"utterance {b}", texts[b], ys[b], Q, "code")
        T = [int(y.shape[0]) for y in ys]
        Tp = [min(int(t * 0.5), 3 * 75) for t in T]
        text_all = torch.cat([t.to(torch.int64) for t in texts]).to(dev)
        prm_all = torch.cat([ys[b][:Tp[b]].to(torch.int64) for b in range(B)]).contiguous().to(dev)
        utts = [_Utt(b, t, pr, Tp[b]) for b, (t, pr) in
                enumerate(zip(text_all.split([int(t.numel()) for t in texts]), prm_all.split(Tp)))]
        codes, cu_g = self._nar(utts, [T[b] - Tp[b] for b in range(B)],
                                torch.cat([ys[b][Tp[b]:, 0].to(torch.int64) for b in range(B)]).to(dev))
        if any(t.is_cuda for t in list(texts) + list(ys)):
            ops.check_oob(dev)
        return [codes[cu_g[b]:cu_g[b + 1]] for b in range(B)]

    def kernel_launches(self) -> int:
        """kernels of libvalle_b200.so executed so far by this process (direct + graph replays)."""
        return int(self.lib.vb_launch_count()) - self.captured_launches + self.replayed_launches

    # ---- helpers ---------------------------------------------------------------------------
    def _embed_pe(self, tokens, tok_stride, table, pe, alpha, n, x, rows, pos, prenet=None):
        """x[rows[r]] = prenet(table[tokens[r*tok_stride]]) + alpha * pe[pos[r]]  (embedding, pre-net, position:
        valle.py:994-997 / 1013-1015); prenet = (name, lengths) of a text pre-net or None (identity)."""
        tmp = torch.empty((n, table.shape[1]), dtype=torch.float32, device=self.device)
        ops.embed_sum(tokens, tok_stride, 0, [table.detach()], n, tmp)
        if prenet is not None:
            tmp = self._text_prenet(tmp, prenet[1], prenet[0])
        ops.add_pe(tmp, pe, alpha.detach(), x, n, positions=pos, out_rows=rows)

    def _replay_steps(self, buf: _ArBuffers, head: L.ArHead, k: int):
        """k decode steps that draw on the device as ONE CUDA graph (captured on first use per (buffer, head tables,
        draw mode, shared prefixes, scores, k))"""
        key = (head.pe, head.predict_w, head.audio_emb, head.greedy, buf.kv_dtype, bool(buf.st.kv_parent),
               bool(buf.st.logprob), buf.st.beam_width, bool(buf.st.beam_first), k)
        graphs = buf.graphs
        ent = graphs.get(key)
        if ent is None:
            if any(kk[:3] != key[:3] for kk in graphs):
                graphs.clear()                      # tables moved: the old captures hold stale pointers
            for _ in range(k):
                self._launch_step(buf, head)        # warm-up launches (function attributes) == these k steps
            g = torch.cuda.CUDAGraph()
            n0 = self.lib.vb_launch_count()
            with torch.cuda.graph(g):
                for _ in range(k):
                    self._launch_step(buf, head)
            kernels = self.lib.vb_launch_count() - n0
            self.captured_launches += kernels
            graphs[key] = (g, kernels, head)        # keep the head struct alive
            return                                  # the warm-up launches were these steps
        ent[0].replay()
        self.replayed_launches += ent[1]

    def _launch_step(self, buf, head: L.ArHead):
        L.check(self.lib.vb_ar_decode_step(self.ar.handle, C.byref(head), C.byref(buf.st), buf.ws.data_ptr(),
                                           buf.ws.numel(), L.stream_ptr()), "vb_ar_decode_step")

    def _sample_push(self, buf: _ArBuffers, head: L.ArHead, top_k: int, temperature: float,
                     forced_step: Optional[torch.Tensor] = None, top_p: float = 1.0):
        """valle.py:1287-1302 topk_sampling with torch's own RNG stream (so a fixed torch seed gives
        the reference's draws), then the stop rule + append on the device."""
        from .models.valle import topk_sampling
        if forced_step is not None:  # teacher forcing (test hook): the given ids instead of a draw
            samp = forced_step.contiguous()
        elif self.sample_on_host:
            host = buf.logits[:, : self.n_vocab].cpu()
            samp = torch.cat([topk_sampling(host[b:b + 1], top_k=top_k, top_p=top_p, temperature=temperature).view(-1)
                              for b in range(host.shape[0])]).to(self.device)
        else:
            samp = topk_sampling(buf.logits[:, : self.n_vocab].clone(), top_k=top_k, top_p=top_p,
                                 temperature=temperature).view(-1).contiguous()
        L.check(self.lib.vb_ar_push_tokens(C.byref(head), C.byref(buf.st), samp.data_ptr(), self.d,
                                           L.stream_ptr()), "vb_ar_push_tokens")

    def _nar(self, utts: Sequence[_Utt], Tg: Sequence[int], first_codes: torch.Tensor,
             forced_codes: Optional[torch.Tensor] = None,
             trace: Optional[dict] = None) -> Tuple[torch.Tensor, np.ndarray]:
        """The NAR stages (valle.py:1059-1137) over utts, packed [text | prompt | generated]: first_codes, int64
        [sum(Tg)], holds the first codebook of the Tg[b] generated frames of every utterance in turn.  Returns the
        codes [sum(Tg), Q], packed the same way, and _offsets(Tg)."""
        m, dev, d, Q = self.model, self.device, self.d_nar, self.Q
        cu_g = _offsets(Tg)
        G = int(cu_g[-1])
        codes = torch.empty((G, Q), dtype=torch.int64, device=dev)
        codes[:, 0] = first_codes
        if Q == 1:
            return codes, cu_g
        B = len(utts)
        pm = self.prefix_mode

        def nar_text(u):   # valle.py:1068-1079: prefix modes 2 / 4 keep the first phoneme and those after the enrolled
            return (u.text[:1], u.text[u.enroll_len - 1:]) if pm in (2, 4) and u.enroll_len is not None else (u.text,)
        pieces = [nar_text(u) for u in utts]
        S2 = [sum(int(t.shape[0]) for t in ps) for ps in pieces]
        text_nar = torch.cat([t for ps in pieces for t in ps])
        prm_all = torch.cat([u.prompt for u in utts])
        Tp = [int(u.prompt.shape[0]) for u in utts]
        T = [Tp[b] + Tg[b] for b in range(B)]
        Ltot = [S2[b] + T[b] for b in range(B)]
        # index maps (host-built with numpy, one H2D)
        cu_np, cut_np = _offsets(Ltot), _offsets(T)
        M, NT = int(cu_np[-1]), int(cut_np[-1])
        S2_np, Tp_np = np.asarray(S2, dtype=np.int64), np.asarray(Tp, dtype=np.int64)
        trow, tpos = _seg_ranges(cu_np[:-1], S2)
        yrow, ypos = _seg_ranges(cu_np[:-1] + S2_np, T)
        y_prompt_rows = _seg_ranges(cut_np[:-1], Tp)[0]
        y_gen_rows = _seg_ranges(cut_np[:-1] + Tp_np, Tg)[0]
        tgt_rows = _seg_ranges(cu_np[:-1] + S2_np + Tp_np, Tg)[0]
        meta = torch.from_numpy(np.concatenate([cu_np, trow, tpos, yrow, ypos, y_prompt_rows, y_gen_rows,
                                                tgt_rows]).astype(np.int32)).to(dev)
        cu_d, trow_d, tpos_d, yrow_d, ypos_d, yp_d, yg_d, tgt_d = meta.split(
            [B + 1, sum(S2), sum(S2), NT, NT, sum(Tp), G, G])

        emb = [e.weight.detach() for e in m.nar_audio_embeddings]
        # y_emb = nar_audio_embeddings[0](y)  (valle.py:1064); rows packed [prompt_b | generated_b]
        y_emb = torch.empty((NT, d), dtype=torch.float32, device=dev)
        ops.embed_sum(prm_all, Q, 0, [emb[0]], sum(Tp), y_emb, out_rows=yp_d)
        ops.embed_sum(codes, Q, 0, [emb[0]], G, y_emb, out_rows=yg_d)
        if pm != 0:  # valle.py:1110-1113: prompt rows get all 8 codebooks up front, in order j=1..7
            ops.embed_sum(prm_all[:, 1:], Q, 1, emb[1:Q], sum(Tp), y_emb, out_rows=yp_d, accumulate=True)
        pe_t = self._pe(m.nar_text_position, max(S2))
        pe_a = self._pe(m.nar_audio_position, max(T))
        ada = self._ada_tables()
        x = torch.empty((M, d), dtype=torch.float32, device=dev)
        logits = torch.empty((G, NUM_AUDIO_TOKENS), dtype=torch.float32, device=dev)
        x_text = None
        if self.pre:   # valle.py:1081-1083: the text side (embedding, pre-net) is computed once for all stages
            x_text = torch.empty((sum(S2), d), dtype=torch.float32, device=dev)
            ops.embed_sum(text_nar, 1, 0, [m.nar_text_embedding.weight.detach()], sum(S2), x_text)
            x_text = self._text_prenet(x_text, S2, "nar_text")
        for i in range(Q - 1):
            # xy_pos = concat([nar_text_position(nar_text_embedding(text)), nar_audio_position(y_emb)])
            if x_text is not None:
                ops.add_pe(x_text, pe_t, m.nar_text_position.alpha.detach(), x, sum(S2), positions=tpos_d, out_rows=trow_d)
            else:
                self._embed_pe(text_nar, 1, m.nar_text_embedding.weight, pe_t, m.nar_text_position.alpha, sum(S2), x, trow_d, tpos_d)
            # valle.py:1092,1121: y_pos = nar_audio_position(nar_audio_prenet(y_emb))
            y_in = self._audio_prenet(y_emb, "nar_audio") if self.pre else y_emb
            ops.add_pe(y_in, pe_a, m.nar_audio_position.alpha.detach(), x, NT, positions=ypos_d, out_rows=yrow_d)
            self.nar.forward(x, cu_d, B, max(Ltot), L.VB_MASK_FULL, None, ada[i])
            hn = self.nar.head_rows(x, ada[i], tgt_d, self.dtype)
            ops.linear(hn, self.nar_predict_w[i], None, L.VB_EPI_NONE, out=logits)
            nxt = emb[i + 1] if i < Q - 2 else None
            if trace is not None:
                trace.setdefault("nar_logits", []).append(logits.clone())
            if forced_codes is not None:  # teacher forcing (test hook): record the argmax, continue with the given ids
                ops.nar_argmax_accumulate(logits, codes[:, i + 1], codes.stride(0), None, None, yg_d)
                if trace is not None:
                    trace.setdefault("nar_argmax", []).append(codes[:, i + 1].clone())
                codes[:, i + 1] = forced_codes[:, i + 1]
                if nxt is not None:
                    ops.embed_sum(codes[:, i + 1:], Q, 0, [nxt], G, y_emb, out_rows=yg_d, accumulate=True)
            else:
                # samples -> codes[:, i+1]; y_emb[generated rows] += emb[i+1][samples]  (valle.py:1130-1134)
                ops.nar_argmax_accumulate(logits, codes[:, i + 1], codes.stride(0), nxt,
                                          y_emb if nxt is not None else None, yg_d)
            if pm == 0 and i < Q - 2:  # valle.py:1104-1107
                ops.embed_sum(prm_all[:, i + 1:], Q, 0, [emb[i + 1]], sum(Tp), y_emb, out_rows=yp_d, accumulate=True)
        return codes, cu_g
