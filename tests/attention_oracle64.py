"""Float64 masked softmax attention, its rounding-error bound and planted keys, for the L x L attention kernels behind
`vb_attention`: the bf16 wgmma flash kernel (`csrc/attention_wgmma.cu`) and the CUDA-core `attn_varlen_simt_kernel`
(`csrc/attention.cu`) in fp32 and bf16.

Everything here is plain torch and runs on whatever device its tensors live on.  `tests/test_attention_oracle64.py`
checks the masks, the bound and the planted keys on the CPU; `tests/test_attention_oracle64_gpu.py` compares the
kernels with `attention64` under `bound`.

Masks.  `visible` builds each mask from the model: VALLE_AR from `oracle.valle_oracle.ar_inference_mask`, PADDED_AR
and PADDED from the key-padding and causal construction of `oracle.valle_oracle.forward_train` (a padded sequence is
[text padded to seg1_start | audio], S text rows and c1 audio rows real).  `row_mask_rule` restates the kernels' own
`RowMask` rule (csrc/kernels.cuh), and the CPU test holds the two equal.

Planted keys.  With random q and k every key carries about 1/L of a row's softmax mass, so a key the kernel skips or a
key it lets through moves the outputs by O(|v| / L): at L = 1025 a whole dropped 64-key tile moves them by less than
2e-2.  `plant` makes chosen keys dominate chosen rows, so that the same mistakes move them by O(|v|):
  - visible beacons: key j at a mask or tile boundary is set so that the first row that must see it puts most of its
    softmax mass on it (for an audio key under the causal masks that row is the diagonal one);
  - forbidden beacons: at every boundary row, the keys just outside its visible intervals -- the first key it must not
    see, the key before each later interval, and key L, row 0 of the next packed sequence -- are set so that they would
    dominate that row if they leaked;
  - one ramp row, the last row with the most keys, whose score maximum rises by 1/2 on every 64-key tile, so that the
    online-softmax rescale runs on every tile.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import torch

from oracle.valle_oracle import ar_inference_mask

MODES = ("full", "valle_ar", "padded_ar", "padded")
KINDS = ("wgmma", "simt_bf16", "simt_f32")     # the kernel paths of vb_attention
HD, BKV, BQ = 64, 64, 128                      # head dim, key tile, query rows of one wgmma CTA
U_BF16, U_F32 = 2.0 ** -8, 2.0 ** -24          # unit roundoffs
SEG1_START = 60                                # the ragged set's padded text length (test_attention_bitwise_gpu.py)


# ----------------------------------------------------------------------------------------------------------- masks
def visible(mode: str, L: int, S: int = 0, c1: int = 0, seg1_start: int = 0) -> torch.Tensor:
    """bool [L, L]: query row r sees key c, from the model's masks (see the module docstring).  A padded sequence
    shorter than seg1_start is the top-left [L, L] block of the mask of text length seg1_start and no audio."""
    if mode == "full":
        return torch.ones(L, L, dtype=torch.bool)
    if mode == "valle_ar":
        assert 0 <= S <= L
        return ~ar_inference_mask(S, L - S)
    assert mode in ("padded_ar", "padded") and 0 <= S <= seg1_start
    x_len, y_len = seg1_start, max(L - seg1_start, 0)
    assert c1 <= y_len
    pad = torch.cat([torch.arange(x_len) >= S, torch.arange(y_len) >= c1])        # make_pad_mask of x_lens | y_lens
    if mode == "padded_ar":
        blocked = ar_inference_mask(x_len, y_len) | pad[None, :]
    else:
        blocked = pad[None, :].expand(x_len + y_len, -1)
    return ~blocked[:L, :L]


def row_mask_rule(mode: str, L: int, S: int = 0, c1: int = 0, seg1_start: int = 0) -> torch.Tensor:
    """bool [L, L] of the kernels' RowMask rule: row r sees key c iff c < lim0 or s1 <= c < hi1, with
    FULL lim0 = L; VALLE_AR lim0 = max(S, r + 1); PADDED_AR lim0 = S, s1 = seg1_start,
    hi1 = seg1_start + clamp(r - seg1_start + 1, 0, c1); PADDED lim0 = S, s1 = seg1_start, hi1 = seg1_start + c1."""
    r = torch.arange(L)[:, None]
    c = torch.arange(L)[None, :]
    if mode == "full":
        return (c < L).expand(L, L)
    if mode == "valle_ar":
        return c < torch.clamp(r + 1, min=S)
    hi1 = seg1_start + (torch.clamp(r - seg1_start + 1, 0, c1) if mode == "padded_ar" else c1)
    return ((c < S) | ((c >= seg1_start) & (c < hi1))).expand(L, L)


def empty_rows_rule(mode: str, L: int, S: int = 0, c1: int = 0, seg1_start: int = 0) -> set:
    """the rows that see no key: only the padded modes without text have any -- PADDED every row when no audio key is
    real either, PADDED_AR the text rows, and every row when no audio key is real"""
    if mode in ("full", "valle_ar") or S > 0:
        return set()
    if c1 == 0:
        return set(range(L))
    return set(range(min(seg1_start, L))) if mode == "padded_ar" else set()


def kv_max(mode: str, L: int, S: int, q_hi: int) -> int:
    """keys [0, kv_max) hold every key the rows below q_hi see (Packed::kv_max)"""
    return max(S, q_hi) if mode == "valle_ar" else L


def drop_last_tile(mode: str, vis: torch.Tensor, S: int) -> torch.Tensor:
    """`vis` as a wgmma kernel that sweeps one key tile too few (n_tiles - 1) would see it: every 128-row block of
    queries loses the keys of the last 64-key tile it reads"""
    L = vis.shape[0]
    out = vis.clone()
    for q0 in range(0, L, BQ):
        n_tiles = -(-kv_max(mode, L, S, min(q0 + BQ, L)) // BKV)
        out[q0:q0 + BQ, (n_tiles - 1) * BKV:] = False
    return out


# ------------------------------------------------------------------------------------------------------- reference
@dataclass
class Ref:
    O: torch.Tensor       # [H, L, 64] float64: softmax(q k^T / 8 + mask) v
    A: torch.Tensor       # [H, L, 64] float64: softmax(...) |v|, what the rounding of P and of the sums scales with
    E: torch.Tensor       # [H, L] float64: bound on the relative error of any p_j of the row (`score_error`)
    empty: set            # rows that see no key (O = A = 0 there)


def attention64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, vis: torch.Tensor, head_chunk: int = 4) -> Ref:
    """masked softmax attention in float64 from the inputs the kernel reads (q, k, v [H, L, 64] of any float dtype,
    already rounded as the kernel rounds them; vis bool [L, L] on the same device).  Heads go `head_chunk` at a time
    so that L = 1500 stays well under 1 GB."""
    H, L, _ = q.shape
    vis = vis.to(q.device)
    empty = set(torch.nonzero(~vis.any(1)).flatten().tolist())
    O, A, E = [], [], []
    for h0 in range(0, H, head_chunk):
        qh, kh, vh = (t[h0:h0 + head_chunk].double() for t in (q, k, v))
        s = (qh @ kh.transpose(-1, -2)) * 0.125
        s = s.masked_fill(~vis, -math.inf)
        m = s.amax(-1, keepdim=True)
        m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
        p = torch.exp(s - m)
        l = p.sum(-1, keepdim=True)
        l = torch.where(l > 0, l, torch.ones_like(l))
        O.append((p @ vh) / l)
        A.append((p @ vh.abs()) / l)
        E.append(score_error(qh, kh, s, m, vis))
    return Ref(torch.cat(O), torch.cat(A), torch.cat(E), empty)


def score_error(q: torch.Tensor, k: torch.Tensor, s: torch.Tensor, m: torch.Tensor, vis: torch.Tensor) -> torch.Tensor:
    """per row, max over its keys of a bound on the relative error of the kernel's p_j = exp(s_j - m) before the
    rescales: the fp32 dot product of 64 terms (gamma_64 sum_i |q_i k_i| / 8, with twice the fp32 unit roundoff
    because the order and rounding of the tensor cores' sums are not specified), the rounded scale and subtraction
    (2^-21 (|s_j| + |m|), several roundings of those magnitudes, in the log2 domain of the wgmma kernel too)"""
    dot = (q.abs() @ k.abs().transpose(-1, -2)) * 0.125
    e = gamma(HD, 2 * U_F32) * dot + 2.0 ** -21 * (s.abs() + m.abs())
    return e.masked_fill(~vis, 0.0).amax(-1)


def gamma(n: int, u: float) -> float:
    return n * u / (1 - n * u)


# ----------------------------------------------------------------------------------------------------------- bound
def bound(ref: Ref, kind: str) -> torch.Tensor:
    """Per-element bound on |o_kernel - o| for the kernel path `kind`, [H, L, 64] float64.

    Write p_j = exp(s_j - m), l = sum_j p_j, o = sum_j p_j v_j / l and a = sum_j p_j |v_j| / l (`Ref.A`).  The
    kernels compute, in fp32 with the key tiles of 64 in order:
      p^_j = p_j (1 + eta_j), |eta_j| <= eps.  The score error `Ref.E`, plus one exp (2 ulp for expf, ex2.approx
          within that) per p_j and one per online-softmax rescale of the row: (T + 1) 2^-21 over T key tiles.
      P:  the wgmma kernel rounds p^_j to bf16 before P V: p~_j = p^_j (1 + rho_j), |rho_j| <= u_P = 2^-8.  The
          row sum l^ is summed from the fp32 p^_j.  The CUDA-core kernels keep fp32 P; the bf16 one still gets
          u_P = 2^-8: its output rounding alone reaches 2^-8 |o|, and the slack keeps a correct kernel at half the
          bound or less even on rows where one key carries all the mass (a = |o|).  The fp32 kernel gets u_P = 0.
      sums:  sum_j p~_j v_j and l^ are fp32 chains of at most n = L + 64 operations (the products, the tile
          rescales o *= corr and l = l corr + rs); each is off by gamma_n (with u = 2^-23 for the tensor cores' sums).
      out:  o^ = fl(fl(N^ * fl(1 / l^))): two fp32 roundings, then the store rounds to the output type, u_out =
          2^-8 for bf16, 2^-24 for fp32.
    Then N^ / l = sum_j p_j v_j (1 + eta_j + rho_j + theta_j) / l, off o by at most (u_P + eps + gamma_n) a, and
    l^ = l (1 + lambda) with |lambda| <= eps + gamma_n moves the quotient by |o| |lambda| to first order, so
        |o^ - o| <= (u_P + eps + gamma_n) a + (u_out + eps + gamma_n + 2^-23) |o|,
    times 1 + 2^-5 for the second-order terms, plus 2^-100 for the p_j that ex2.approx.ftz flushes to zero.  For the
    bf16 kernels this is about 2^-8 (a + |o|); for the fp32 kernel about gamma_{L+64} (a + |o|).  The rounding error
    actually made is a sum of many independent roundings, so it stays a fraction of this worst case."""
    L = ref.O.shape[1]
    T = -(-L // BKV)
    g = gamma(L + 64, 2 * U_F32)
    eps = ref.E[..., None] + (T + 1) * 2.0 ** -21
    u_p = 0.0 if kind == "simt_f32" else U_BF16
    u_out = U_F32 if kind == "simt_f32" else U_BF16
    b = (u_p + eps + g) * ref.A + (u_out + eps + g + 2 * U_F32) * ref.O.abs()
    return b * (1 + 2.0 ** -5) + 2.0 ** -100


def ratio(got: torch.Tensor, ref: Ref, bnd: torch.Tensor) -> float:
    """max |got - O| / bound over the rows that see a key (got [H, L, 64]); a NaN or inf there counts as infinite"""
    keep = torch.ones(got.shape[1], dtype=torch.bool)
    if ref.empty:
        keep[list(ref.empty)] = False
    keep = keep.to(got.device)
    d = (got.double() - ref.O)[:, keep]
    r = d.abs() / bnd[:, keep]
    r = torch.where(torch.isfinite(d), r, torch.full_like(r, math.inf))
    return float(r.max()) if r.numel() else 0.0


# -------------------------------------------------------------------------------------------------------- backward
def _probs(q, k, vis):
    s = (q @ k.transpose(-1, -2)) * 0.125
    s = s.masked_fill(~vis, -math.inf)
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    return s, m, p / torch.where(l > 0, l, torch.ones_like(l)), m + torch.log(torch.where(l > 0, l, torch.ones_like(l)))


def attention_bwd64(q, k, v, o, dO, vis, w=None, head_chunk: int = 4):
    """(dq, dk, dv) [H, L, 64] float64 of O = (P o w) V, P = softmax(q k^T / 8 + mask), for the output gradient dO:
    dV = (P o w)^T dO, dP = w o (dO V^T), D = rowsum(dO o o), dS = P o (dP - D), dQ = dS K / 8, dK = dS^T Q / 8.
    D is formed from the `o` given; w: the dropout scale [H, L, L] (None: no dropout)."""
    H = q.shape[0]
    out = ([], [], [])
    for h0 in range(0, H, head_chunk):
        sl = slice(h0, h0 + head_chunk)
        qh, kh, vh, oh, gh = (t[sl].double() for t in (q, k, v, o, dO))
        _, _, P, _ = _probs(qh, kh, vis)
        Pw = P if w is None else P * w[sl]
        dP = gh @ vh.transpose(-1, -2)
        if w is not None:
            dP = dP * w[sl]
        dS = P * (dP - (gh * oh).sum(-1, keepdim=True))
        out[0].append(dS @ kh * 0.125)
        out[1].append(dS.transpose(-1, -2) @ qh * 0.125)
        out[2].append(Pw.transpose(-1, -2) @ gh)
    return tuple(torch.cat(t) for t in out)


def bwd_bound(q, k, v, o_st, dO, vis, w=None, head_chunk: int = 4):
    """(exact, bound) for dq, dk, dv of `attn_bwd_dq_kernel` / `attn_bwd_dkv_kernel` (csrc/backward.cu), each
    [H, L, 64] float64, from the inputs the kernels read: q, k, v [H, L, 64], the stored output o_st and dO (all
    already rounded as stored) and the dropout scale w [H, L, L] (None: none).  `exact` is the true
    gradient: attention_bwd64 with D formed from the float64 output O = (P o w) V, not from o_st.

    The kernels, in fp32 over 64 x 64 tiles, sums as fmaf chains in order (u = 2^-24; the score and product sums
    get 2u, as `score_error`):
      p:   p^ = expf(s^ / 8 - lse^) = P (1 + eta).  The score error E (`score_error`), lse = m + logf(l) from the
           online sweep: l is off by gamma_{L+64}, logf adds 2^-23, the sum m + log l one u |lse|; s / 8 - lse one u
           (|s / 8| + |lse|) and expf 2^-22: eta <= E + gamma_{L+64}(2u) + 2^-21 (|s / 8| + |lse| + 2).
      dP:  dP^ = dP + e, |e| <= gamma_64(2u) |dO| |V|^T; the dropout scale one more u |w dP|.
      D:   D^ = rowsum(dO o o_st) in 16-term chains and two shuffle adds: |D^ - D| <= gamma_64(2u) rowsum |dO| |o_st|
           + rowsum |dO| |o_st - O|, the second the stored output's own rounding, which D inherits.
      dS:  fl(p^ fl(dP^ - D^)): the errors above are absolute, so the cancellation in dP - D costs nothing extra:
           |dS^ - dS| <= P (|e| + u |w dP| + |D^ - D|) + (eta + 2u) P |w dP - D| =: e_S.
      sums: dQ = sum over key tiles of dS K (one fmaf chain of kv_max <= L terms), dK over query tiles (L terms):
           |dQ^ - dQ| <= (e_S |K| + gamma_{L+64}(u) |dS| |K|) / 8, dK the same with dS^T and |Q|;
           dV = sum_q fl(p^ w) dO: |dV^ - dV| <= ((eta + u) P w)^T |dO| + gamma_{L+64}(u) (P w)^T |dO|.
      out: the scale by 1/8 is exact; a bf16 store adds half_ulp(out), which the caller adds
           (stack_oracle64.attn_bwd_ratio), as it has the output.
    Bound: the first-order sum times 1 + 2^-5, + 2^-120.  A key no query sees and a query that sees no key get a
    bound of 2^-120 (+ the half ulp of 0): their gradient rows must be exactly 0."""
    H, L, _ = q.shape
    u, g64 = U_F32, gamma(HD, 2 * U_F32)
    gL = gamma(L + 64, 2 * U_F32)
    ex, bd = ([], [], []), ([], [], [])
    for h0 in range(0, H, head_chunk):
        sl = slice(h0, h0 + head_chunk)
        qh, kh, vh, oh, gh = (t[sl].double() for t in (q, k, v, o_st, dO))
        s, m, P, lse = _probs(qh, kh, vis)
        E = score_error(qh, kh, s, m, vis)[..., None]
        ww = torch.ones_like(P) if w is None else w[sl].double()
        Pw = P * ww
        O = Pw @ vh
        dP = gh @ vh.transpose(-1, -2)
        D = (gh * O).sum(-1, keepdim=True)
        wdP = ww * dP
        dS = P * (wdP - D)
        sfin = torch.where(vis, s.abs(), torch.zeros_like(s))
        eta = E + gL + 2.0 ** -21 * (sfin + lse.abs() + 2)
        e_dp = g64 * (gh.abs() @ vh.abs().transpose(-1, -2)) * ww + u * wdP.abs()
        e_D = g64 * (gh.abs() * oh.abs()).sum(-1, keepdim=True) + (gh.abs() * (oh - O).abs()).sum(-1, keepdim=True)
        e_S = P * (e_dp + e_D) + (eta + 2 * u) * P * (wdP - D).abs()
        ex[0].append(dS @ kh * 0.125)
        ex[1].append(dS.transpose(-1, -2) @ qh * 0.125)
        ex[2].append(Pw.transpose(-1, -2) @ gh)
        aS = dS.abs()
        bd[0].append((e_S @ kh.abs() + gL * aS @ kh.abs()) * 0.125)
        bd[1].append((e_S.transpose(-1, -2) @ qh.abs() + gL * aS.transpose(-1, -2) @ qh.abs()) * 0.125)
        bd[2].append((((eta + u) * Pw).transpose(-1, -2) + gL * Pw.transpose(-1, -2)) @ gh.abs())
    exact = tuple(torch.cat(t) for t in ex)
    return exact, tuple(torch.cat(b) * (1 + 2.0 ** -5) + 2.0 ** -120 for b in bd)


def emulate_bwd(q, k, v, o, dO, vis, w=None, out_dtype=torch.float32, skip_last_q_tile=False,
                skip_last_k_tile=False, d_dims=HD, drop_dp=True):
    """the arithmetic of attn_bwd_dq_kernel / attn_bwd_dkv_kernel in fp32 on the stored inputs (q, k, v, o, dO
    [H, L, 64] of the storage dtype): lse by the online sweep over 64-key tiles, D = rowsum(dO o o) in fp32, p =
    exp(s / 8 - lse), dS = p (w dP - D), dQ summed over key tiles in order, dK / dV over query tiles in order, then
    the store.  The keyword arguments plant mistakes: dK / dV skipping the last partial query tile, dQ skipping the
    last key tile, D over the first d_dims head dims, the dropout scale on P but not on dP (drop_dp=False)."""
    H, L, _ = q.shape
    qf, kf, vf, of, gf = (t.float() for t in (q, k, v, o, dO))
    s = (qf @ kf.transpose(-1, -2)) * 0.125
    s = s.masked_fill(~vis, -math.inf)
    m = torch.full((H, L), -math.inf)
    l = torch.zeros(H, L)
    for j0 in range(0, L, BKV):
        t = s[..., j0:j0 + BKV]
        mn = torch.maximum(m, t.amax(-1))
        mu = torch.where(mn == -math.inf, torch.zeros_like(mn), mn)
        l = l * torch.exp(m - mu) + torch.exp(t - mu[..., None]).sum(-1)
        m = mn
    lse = torch.where(l > 0, m + torch.log(l), torch.full_like(l, math.inf))
    D = (gf[..., :d_dims] * of[..., :d_dims]).sum(-1, keepdim=True)
    p = torch.exp(s - lse[..., None])
    dP = gf @ vf.transpose(-1, -2)
    wf = torch.ones(H, L, L) if w is None else w.float()
    dS = p * ((dP * wf if drop_dp else dP) - D)
    pw = p * wf
    dq = torch.zeros(H, L, HD)
    n_kt = -(-L // BKV)
    for j0 in range(0, L, BKV):
        if skip_last_k_tile and j0 // BKV == n_kt - 1 and n_kt > 1:
            break
        dq = dq + dS[..., j0:j0 + BKV] @ kf[:, j0:j0 + BKV]
    dk, dv = torch.zeros(H, L, HD), torch.zeros(H, L, HD)
    for q0 in range(0, L, BKV):
        if skip_last_q_tile and q0 + BKV > L:
            break
        dk = dk + dS[:, q0:q0 + BKV].transpose(-1, -2) @ qf[:, q0:q0 + BKV]
        dv = dv + pw[:, q0:q0 + BKV].transpose(-1, -2) @ gf[:, q0:q0 + BKV]
    return tuple((t * (0.125 if i < 2 else 1.0)).to(out_dtype) for i, t in enumerate((dq, dk, dv)))


# ------------------------------------------------------------------------------------------------------- emulation
def emulate(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, vis: torch.Tensor, kind: str) -> torch.Tensor:
    """the arithmetic of one kernel path in float32 / bf16 on the rounded inputs (q, k, v [H, L, 64] float32): 64-key
    tiles in order, fp32 scores, masked online softmax with the running maximum (exp2 of the log2-scaled scores for
    the wgmma kernel, exp for the CUDA-core kernels), P rounded to bf16 before P V on the wgmma path, the output
    rounded to bf16 on the bf16 paths.  Not bit-exact (the sums go in torch's order), but rounded where the kernels
    round; returns [H, L, 64] float32."""
    H, L, _ = q.shape
    wg = kind == "wgmma"
    sc = torch.tensor(0.125 * 1.4426950408889634 if wg else 0.125, dtype=torch.float32)
    ex = torch.exp2 if wg else torch.exp
    o = torch.zeros(H, L, HD)
    m = torch.full((H, L), -math.inf)
    l = torch.zeros(H, L)
    for j0 in range(0, L, BKV):
        s = (q @ k[:, j0:j0 + BKV].transpose(-1, -2)) * sc
        s = s.masked_fill(~vis[:, j0:j0 + BKV], -math.inf)
        mn = torch.maximum(m, s.amax(-1))
        mu = torch.where(mn == -math.inf, torch.zeros_like(mn), mn)
        corr = ex(m - mu)
        p = ex(s - mu[..., None])
        l = l * corr + p.sum(-1)
        pv = p.bfloat16().float() if wg else p
        o = o * corr[..., None] + pv @ v[:, j0:j0 + BKV]
        m = mn
    out = o * (1.0 / l)[..., None]
    return out if kind == "simt_f32" else out.bfloat16().float()


# -------------------------------------------------------------------------------------------------- planted keys
@dataclass
class Beacon:
    seq: int
    kind: str             # "visible" or "forbidden"
    row: int              # the query row (of sequence `seq`) the key is aimed at
    key: int              # key index counted from the start of sequence `seq`; L is row 0 of the next sequence


@dataclass
class Batch:
    """a packed batch for vb_attention: qkv [M, 3 H 64] float32 (the fp32 kernel's input; the bf16 paths read it
    rounded), and per sequence its length, text length S and real audio length c1"""
    name: str
    qkv: torch.Tensor
    lens: List[int]
    mode: str
    S: List[int]
    c1: List[int]
    seg1_start: int
    H: int
    beacons: List[Beacon] = field(default_factory=list)

    @property
    def cu(self) -> List[int]:
        c = [0]
        for n in self.lens:
            c.append(c[-1] + n)
        return c

    def vis(self, b: int) -> torch.Tensor:
        return visible(self.mode, self.lens[b], self.S[b], self.c1[b], self.seg1_start)

    def heads(self, qkv: torch.Tensor, b: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """q, k, v [H, L, 64] of sequence b from qkv [M, 3 H 64] (any dtype)"""
        r0, n, D = self.cu[b], self.lens[b], self.H * HD
        blk = qkv[r0:r0 + n]
        return tuple(blk[:, i * D:(i + 1) * D].reshape(n, self.H, HD).transpose(0, 1) for i in range(3))


def boundary_positions(L: int, S: int, c1: int, seg1_start: int, mode: str) -> List[int]:
    """key / row positions where tiles or mask intervals start and end"""
    pos = {0, 63, 64, 127, 128, 191, 192, L - 2, L - 1}
    if mode != "full":
        pos |= {S - 1, S}
    if mode.startswith("padded"):
        pos |= {seg1_start - 1, seg1_start, seg1_start + c1 - 1, seg1_start + c1}
    return sorted(p for p in pos if 0 <= p < L)


def forbidden_keys(vis_row: torch.Tensor) -> List[int]:
    """the keys just outside each visible interval of one row: the first key past each interval, the key before each
    interval but the first (key L, past the last key, stands for row 0 of the next sequence)"""
    f = torch.zeros(1, dtype=torch.bool)
    prev, nxt = torch.cat([f, vis_row[:-1]]), torch.cat([vis_row[1:], f])
    ends = torch.nonzero(vis_row & ~nxt).flatten() + 1
    starts = torch.nonzero(vis_row & ~prev).flatten() - 1
    return sorted(set(ends.tolist()) | set(s for s in starts.tolist() if s >= 0))


def plant(batch: Batch, gen: torch.Generator, strength: float = 4.0, ramp: float = 0.5) -> None:
    """Plant the beacons of the module docstring into batch.qkv (in place) and list them in batch.beacons.  A beacon
    aimed at row r adds (8 T / |q_r|^2) q_r to its key, so that q_r . k / 8 gains T = ln(keys row r sees) + strength
    (the key then carries most of the row's mass), in every head; its value row becomes 2 N(0, 1).  Keys aimed at
    by several beacons carry the sum."""
    qkv, H = batch.qkv, batch.H
    D = H * HD
    cu, B = batch.cu, len(batch.lens)
    dev = qkv.device
    planted = set()                                     # packed rows whose value row was replaced
    for b in range(B):
        L, S, c1 = batch.lens[b], batch.S[b], batch.c1[b]
        vis = batch.vis(b)
        n_vis = vis.sum(1)
        q, k, v = (qkv[cu[b]:cu[b] + L, i * D:(i + 1) * D].view(L, H, HD) for i in range(3))
        rows_used = set()
        if ramp > 0 and L > BKV and bool(n_vis.any()):
            r = int(L - 1 - torch.argmax(n_vis.flip(0)))   # the last row with the most keys
            rows_used.add(r)
            qr = q[r]                                     # [H, 64]
            keys = torch.nonzero(vis[r]).flatten()
            t = (keys // BKV).to(qkv.dtype).to(dev) * ramp
            k[keys.to(dev)] += (8.0 * t[:, None, None] / (qr * qr).sum(-1)[None, :, None]) * qr[None]
        pos = boundary_positions(L, S, c1, batch.seg1_start, batch.mode)
        aims = []
        for j in pos:                                   # visible beacons
            rows = [int(x) for x in torch.nonzero(vis[:, j]).flatten().tolist() if int(x) not in rows_used]
            if rows:
                rows_used.add(rows[0])
                aims.append(Beacon(b, "visible", rows[0], j))
        for r in pos:                                   # forbidden beacons
            if n_vis[r] == 0:
                continue
            for j in forbidden_keys(vis[r]):
                if j < L or b + 1 < B:
                    aims.append(Beacon(b, "forbidden", r, j))
        for bc in aims:
            kr = cu[b] + bc.key                          # packed row of the key (row 0 of b + 1 for key L)
            qr = q[bc.row]
            T = math.log(max(int(n_vis[bc.row]), 1)) + strength
            qkv[kr, D:2 * D].view(H, HD).add_((8.0 * T / (qr * qr).sum(-1))[:, None] * qr)
            if kr not in planted:
                planted.add(kr)
                qkv[kr, 2 * D:] = 2.0 * torch.randn(D, generator=gen).to(dev)
        batch.beacons.extend(aims)


def beacon_vis(vis: torch.Tensor, bc: Beacon) -> torch.Tensor:
    """row bc.row of `vis` with the beacon's key omitted (visible) or let through (forbidden), over keys [0, L + 1)"""
    row = torch.cat([vis[bc.row], torch.zeros(1, dtype=torch.bool)])
    row[bc.key] = bc.kind == "forbidden"
    return row


# ----------------------------------------------------------------------------------------------------------- cases
SWEEP_L = (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 256, 257)


def _sweep_seqs(mode: str, seg1_start: int):
    """(L, S, c1) of the packed length sweep: S in {1, 63, 64, 65, L}, and in the padded modes S <= seg1_start
    (0 included: rows without keys) and c1 in {0, 1, 64, L - seg1_start}"""
    out = []
    for L in SWEEP_L:
        if mode == "full":
            out.append((L, 0, 0))
        elif mode == "valle_ar":
            out += [(L, S, 0) for S in sorted({1, 63, 64, 65, L}) if S <= L]
        else:
            y = max(L - seg1_start, 0)
            out += [(L, S, c) for S in sorted({0, 1, 63, 64, 65, L}) if S <= min(L, seg1_start)
                    for c in sorted({0, 1, 64, y}) if c <= y]
    return out


def _ragged_lengths():
    """the 28 sequences of test_attention_bitwise_gpu._ragged: 1-row and 1-key remainders, 1 to 400 rows"""
    g = torch.Generator().manual_seed(11)
    B = 28
    lens = [1, 129, 257, 400, 128, 256, 385] + torch.randint(2, 400, (B - 7,), generator=g).tolist()
    S = [min(n, int(v)) for n, v in zip(lens, torch.randint(1, 60, (B,), generator=g).tolist())]
    seg1 = [max(0, min(n - SEG1_START, int(v))) for n, v in zip(lens, torch.randint(0, 340, (B,), generator=g).tolist())]
    return lens, S, seg1


def case_names() -> List[str]:
    names = ["nar_b64_l1025", "prefill_b64_l272"]
    names += [f"config2_b4_l1500_{m}" for m in MODES]
    names += [f"ragged_{m}" for m in MODES]
    names += ["sweep_full", "sweep_valle_ar"]
    names += [f"sweep_{m}_s{s}" for m in ("padded_ar", "padded") for s in (1, 64, 65)]
    return names


def make_case(name: str, device="cpu", B: Optional[int] = None, H: Optional[int] = None) -> Batch:
    """the seeded, planted batch `name` (case_names()); B / H cut the sequences and heads (the CPU tests run smaller
    copies of the GPU cases).  Random numbers are drawn on the CPU, so every device gets the same batch."""
    seed = sum(ord(c) for c in name)
    gen = torch.Generator().manual_seed(seed)
    seg1_start, scale, peaked = 0, 0.5, False
    if name == "nar_b64_l1025":                 # the benchmark's NAR passes
        mode, hh, lens, S, c1, peaked = "full", 16, [1025] * 64, [0] * 64, [0] * 64, True
    elif name == "prefill_b64_l272":            # the benchmark's AR prefill: 47 text + 225 prompt rows
        mode, hh, lens, S, c1 = "valle_ar", 16, [272] * 64, [47] * 64, [0] * 64
    elif name.startswith("config2_"):           # L % 64 = 28, L % 128 = 92
        mode, hh, seg1_start = name[len("config2_b4_l1500_"):], 16, 150
        lens, S, c1 = [1500] * 4, [47, 150, 1, 100], [1350, 700, 1, 0]
    elif name.startswith("ragged_"):
        mode, hh, seg1_start, scale = name[len("ragged_"):], 16, SEG1_START, 0.7
        lens, S, c1 = _ragged_lengths()
        if mode == "full":
            S = [0] * len(lens)
        if not mode.startswith("padded"):
            c1 = [0] * len(lens)
    else:
        rest = name[len("sweep_"):]
        mode, seg1_start = (rest.rsplit("_s", 1)[0], int(rest.rsplit("_s", 1)[1])) if "_s" in rest else (rest, 0)
        hh = 4
        lens, S, c1 = (list(x) for x in zip(*_sweep_seqs(mode, seg1_start)))
    if B is not None:
        lens, S, c1 = lens[:B], S[:B], c1[:B]
    hh = H or hh
    qkv = torch.randn(sum(lens), 3 * hh * HD, generator=gen) * scale
    if peaked:                                  # sequence 0's scores x 6: its row maxima move late in the sweep
        qkv[:lens[0], :hh * HD] *= 6.0
    batch = Batch(name, qkv.to(device), lens, mode, S, c1, seg1_start, hh)
    plant(batch, gen)
    return batch
