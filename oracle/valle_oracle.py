"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference VALL-E hot path.

This file is the *oracle* for the sm_90a engine in `valle_b200/`.  It restates,
in explicit torch-CPU fp32 arithmetic on a plain `state_dict`, what
lifeiteng/vall-e computes in

  * valle/models/valle.py:961-1137   VALLE.inference (AR loop + 7 NAR passes)
  * valle/models/valle.py:1139-1238  VALLE.continual
  * valle/models/valle.py:762-959    VALLE.forward   (training loss/metrics)
  * valle/models/valle.py:1242-1302  top_k_top_p_filtering / topk_sampling
  * valle/modules/transformer.py:57-108,265-334,363-406 (LayerNorm, AdaptiveLayerNorm,
    TransformerEncoderLayer pre-LN, TransformerEncoder + final norm)
  * valle/modules/activation.py:199-431 -> F.multi_head_attention_forward
  * valle/modules/embedding.py:68-97 (sine PE table, x + alpha*pe)

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import it -- as the checker or the timed CPU
baseline, never as part of the product path.  The product (`valle_b200`) must
fail loudly without its CUDA library and never routes through this file.

PINNING: the reference's own tests hold no golden vectors for this path
(SURVEY.md section 4/8c: valle/tests/valle_test.py is unseeded smoke testing).  The
oracle is therefore pinned against *outputs of the reference itself run in the
build container* (`oracle/ref_loader.py` exec's the unmodified files):
`tests/test_oracle.py` compares every function here with the real
classes whenever /root/reference is mounted, and `oracle/gen_golden.py` writes
reference-generated fixtures to `tests/golden/` that travel to the GPU box.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

NUM_TEXT_TOKENS = 512    # valle/models/macros.py:2
NUM_AUDIO_TOKENS = 1024  # valle/models/macros.py:5


@dataclass
class OracleConfig:
    d_model: int = 1024
    nhead: int = 16
    num_layers: int = 12
    prefix_mode: int = 0
    num_quantizers: int = 8
    # the north-star path: norm_first=True, add_prenet=False, nar_scale_factor=1.0,
    # prepend_bos=False (valle/models/__init__.py:25-95 defaults)


# --------------------------------------------------------------------------
# operators
# --------------------------------------------------------------------------
def sine_pe(n: int, d: int) -> torch.Tensor:
    """valle/modules/embedding.py:75-91 -- fp32 sin/cos table built on the CPU."""
    pe = torch.zeros(n, d)
    position = torch.arange(0, n, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(
        torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def pos_embed(x: torch.Tensor, alpha: torch.Tensor, start: int = 0) -> torch.Tensor:
    """embedding.py:93-97 with scale=False (x_scale = 1): x + alpha * pe[:, :T]."""
    T, d = x.shape[-2], x.shape[-1]
    pe = sine_pe(start + T, d)[start:]
    return x * 1.0 + alpha * pe


def layer_norm(x, w, b, eps: float = 1e-5):
    """transformer.py:57-74 -> F.layer_norm: biased variance, affine."""
    mu = x.mean(dim=-1, keepdim=True)
    var = ((x - mu) ** 2).mean(dim=-1, keepdim=True)
    return (x - mu) * torch.rsqrt(var + eps) * w + b


def ada_layer_norm(x, stage_emb, proj_w, proj_b, ln_w, ln_b, eps: float = 1e-5):
    """transformer.py:93-108: (weight | bias) = split(Linear(d->2d)(emb)); weight*LN(x)+bias."""
    d = x.shape[-1]
    wb = F.linear(stage_emb, proj_w, proj_b)  # [1, 2d]
    weight, bias = wb[..., :d], wb[..., d:]
    return weight * layer_norm(x, ln_w, ln_b, eps) + bias


def mha(x, in_w, in_b, out_w, out_b, nhead: int,
        blocked: Optional[torch.Tensor] = None,
        key_padding: Optional[torch.Tensor] = None):
    """activation.py:408-427 -> torch.nn.functional.multi_head_attention_forward:
    packed in-proj rows [0:d]=Q [d:2d]=K [2d:3d]=V, heads = contiguous 64-column slices,
    scale 1/sqrt(hd), boolean mask True => -inf, softmax fp32, out-proj with bias.
    x: [B, L, d]; blocked: bool [L, L] or [B*H, L, L] float(-inf) ; key_padding: bool [B, L]."""
    B, L, d = x.shape
    hd = d // nhead
    qkv = F.linear(x, in_w, in_b)
    q, k, v = qkv[..., :d], qkv[..., d:2 * d], qkv[..., 2 * d:]
    q = q.view(B, L, nhead, hd).transpose(1, 2)
    k = k.view(B, L, nhead, hd).transpose(1, 2)
    v = v.view(B, L, nhead, hd).transpose(1, 2)
    s = torch.matmul(q, k.transpose(-1, -2)) * (1.0 / math.sqrt(hd))  # [B,H,L,L]
    if blocked is not None:
        if blocked.dtype == torch.bool:
            s = s.masked_fill(blocked, float("-inf"))
        else:
            s = s + blocked.view(B, nhead, L, L)
    if key_padding is not None:
        s = s.masked_fill(key_padding[:, None, None, :], float("-inf"))
    p = torch.softmax(s, dim=-1)
    o = torch.matmul(p, v).transpose(1, 2).reshape(B, L, d)
    return F.linear(o, out_w, out_b)


def _layer_keys(prefix: str, i: int) -> str:
    return f"{prefix}.layers.{i}."


def encoder(sd: Dict[str, torch.Tensor], prefix: str, x: torch.Tensor, cfg: OracleConfig,
            blocked=None, key_padding=None, stage_emb: Optional[torch.Tensor] = None):
    """transformer.py:363-406 (stack + final norm) over transformer.py:296-302 (pre-LN layer)."""
    adaptive = stage_emb is not None
    for i in range(cfg.num_layers):
        p = _layer_keys(prefix, i)
        if adaptive:
            h = ada_layer_norm(x, stage_emb, sd[p + "norm1.project_layer.weight"],
                               sd[p + "norm1.project_layer.bias"],
                               sd[p + "norm1.norm.weight"], sd[p + "norm1.norm.bias"])
        else:
            h = layer_norm(x, sd[p + "norm1.weight"], sd[p + "norm1.bias"])
        x = x + mha(h, sd[p + "self_attn.in_proj_weight"], sd[p + "self_attn.in_proj_bias"],
                    sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"],
                    cfg.nhead, blocked, key_padding)
        if adaptive:
            h = ada_layer_norm(x, stage_emb, sd[p + "norm2.project_layer.weight"],
                               sd[p + "norm2.project_layer.bias"],
                               sd[p + "norm2.norm.weight"], sd[p + "norm2.norm.bias"])
        else:
            h = layer_norm(x, sd[p + "norm2.weight"], sd[p + "norm2.bias"])
        # _ff_block transformer.py:332-334, activation = ReLU (transformer.py:187)
        x = x + F.linear(F.relu(F.linear(h, sd[p + "linear1.weight"], sd[p + "linear1.bias"])),
                         sd[p + "linear2.weight"], sd[p + "linear2.bias"])
    if adaptive:
        x = ada_layer_norm(x, stage_emb, sd[prefix + ".norm.project_layer.weight"],
                           sd[prefix + ".norm.project_layer.bias"],
                           sd[prefix + ".norm.norm.weight"], sd[prefix + ".norm.norm.bias"])
    else:
        x = layer_norm(x, sd[prefix + ".norm.weight"], sd[prefix + ".norm.bias"])
    return x


def ar_inference_mask(S: int, t: int) -> torch.Tensor:
    """valle.py:1010-1033: bool [S+t, S+t], True = blocked.  Text rows see all text and no
    audio; audio rows see all text and causal audio."""
    x_mask = F.pad(torch.zeros((S, S), dtype=torch.bool), (0, t), value=True)
    y_mask = F.pad(torch.triu(torch.ones(t, t, dtype=torch.bool), diagonal=1), (S, 0), value=False)
    return torch.concat([x_mask, y_mask], dim=0)


def top_k_top_p_filtering(logits, top_k=0, top_p=1.0, filter_value=-float("inf"),
                          min_tokens_to_keep=1):
    """valle.py:1242-1284 (top_p is always 1.0 on this path)."""
    if top_k > 0:
        top_k = min(max(top_k, min_tokens_to_keep), logits.size(-1))
        kth = torch.topk(logits, top_k)[0][..., -1, None]
        logits = logits.masked_fill(logits < kth, filter_value)  # ties keep extras (:1259)
    assert top_p >= 1.0
    return logits


def topk_sampling(logits, top_k=10, top_p=1.0, temperature=1.0, generator=None):
    """valle.py:1287-1302."""
    if temperature != 1.0:
        logits = logits / temperature
    logits = top_k_top_p_filtering(logits, top_k=top_k, top_p=top_p)
    return torch.multinomial(F.softmax(logits, dim=-1), num_samples=1, generator=generator)


# --------------------------------------------------------------------------
# VALLE.inference -- faithful full-recompute restatement
# --------------------------------------------------------------------------
@dataclass
class InferenceTrace:
    ar_logits: List[torch.Tensor]            # one [1025] per AR iteration (incl. the stopping one)
    ar_margin: List[float]                   # top1 - top2 per AR iteration
    nar_logits: List[torch.Tensor]           # 7 x [Tgen, 1024]
    nar_margin: List[torch.Tensor]           # 7 x [Tgen]


def _margin(logits: torch.Tensor) -> torch.Tensor:
    t2 = torch.topk(logits, 2, dim=-1)[0]
    return t2[..., 0] - t2[..., 1]


def inference(sd: Dict[str, torch.Tensor], cfg: OracleConfig, x: torch.Tensor,
              x_lens: torch.Tensor, y: torch.Tensor, enroll_x_lens: Optional[torch.Tensor] = None,
              top_k: int = -100, temperature: float = 1.0, trace: Optional[InferenceTrace] = None,
              max_new_tokens: Optional[int] = None, quiet: bool = True) -> torch.Tensor:
    """valle.py:961-1137.  B == 1 (valle.py:989).  Recomputes the whole text+audio
    sequence per generated token exactly as the reference does (valle.py:1004 TODO)."""
    assert x.ndim == 2 and x_lens.ndim == 1 and y.ndim == 3 and y.shape[0] == 1
    assert torch.all(x_lens > 0)
    d = cfg.d_model
    text = x
    S = int(x_lens.max())
    xe = pos_embed(sd["ar_text_embedding.word_embeddings.weight"][text],
                   sd["ar_text_position.alpha"])
    prompts = y
    Tp = y.shape[1]
    yy = prompts[..., 0]
    while True:
        y_pos = pos_embed(sd["ar_audio_embedding.word_embeddings.weight"][yy],
                          sd["ar_audio_position.alpha"])
        xy = torch.concat([xe, y_pos], dim=1)
        blocked = ar_inference_mask(S, yy.shape[1])
        dec = encoder(sd, "ar_decoder", xy, cfg, blocked=blocked)
        logits = F.linear(dec[:, -1], sd["ar_predict_layer.weight"])  # [1,1025], no bias (:153-155)
        if trace is not None:
            trace.ar_logits.append(logits[0].clone())
            trace.ar_margin.append(float(_margin(logits[0])))
        samples = topk_sampling(logits.clone(), top_k=top_k, top_p=1.0, temperature=temperature)
        n_new = yy.shape[1] - Tp
        if (torch.argmax(logits, dim=-1)[0] == NUM_AUDIO_TOKENS
                or samples[0, 0] == NUM_AUDIO_TOKENS
                or n_new > int(x_lens.max()) * 16
                or (max_new_tokens is not None and n_new >= max_new_tokens)):
            if Tp == yy.shape[1]:
                raise SyntaxError("well trained model shouldn't reach here.")  # valle.py:1049-1052
            if not quiet:
                print(f"VALL-E EOS [{Tp} -> {yy.shape[1]}]")
            break
        yy = torch.concat([yy, samples], dim=1)

    codes = [yy[:, Tp:]]
    if cfg.num_quantizers == 1:
        return torch.stack(codes, dim=-1)
    codes += nar_decode(sd, cfg, text, S, yy, prompts, Tp, enroll_x_lens, trace)
    assert len(codes) == cfg.num_quantizers
    return torch.stack(codes, dim=-1)


def nar_decode(sd, cfg: OracleConfig, text, text_len: int, yy, prompts, Tp: int,
               enroll_x_lens=None, trace: Optional[InferenceTrace] = None,
               trim_text: bool = True) -> List[torch.Tensor]:
    """valle.py:1063-1134 (shared by inference and continual :1180-1235)."""
    Q = cfg.num_quantizers
    y_emb = sd["nar_audio_embeddings.0.word_embeddings.weight"][yy].clone()
    if cfg.prefix_mode in (2, 4) and trim_text:  # valle.py:1068-1079 (inference only)
        enrolled_len = int(enroll_x_lens.max())
        text = torch.concat([text[:, :1], text[:, enrolled_len - 1:]], dim=1)
        text_len = text_len - (enrolled_len - 2)
    xe = pos_embed(sd["nar_text_embedding.word_embeddings.weight"][text],
                   sd["nar_text_position.alpha"])
    out = []
    if cfg.prefix_mode != 0:  # valle.py:1110-1113
        for j in range(1, Q):
            y_emb[:, :Tp] += sd[f"nar_audio_embeddings.{j}.word_embeddings.weight"][prompts[..., j]]
    for i in range(Q - 1):
        y_pos = pos_embed(y_emb, sd["nar_audio_position.alpha"])
        xy = torch.concat([xe, y_pos], dim=1)
        stage = sd[f"nar_stage_embeddings.{i}.word_embeddings.weight"]  # [1, d]
        dec = encoder(sd, "nar_decoder", xy, cfg, stage_emb=stage)
        logits = F.linear(dec[:, text_len + Tp:], sd[f"nar_predict_layers.{i}.weight"])
        samples = torch.argmax(logits, dim=-1)
        if trace is not None:
            trace.nar_logits.append(logits[0].clone())
            trace.nar_margin.append(_margin(logits[0]))
        out.append(samples)
        if i < Q - 2:
            emb = sd[f"nar_audio_embeddings.{i + 1}.word_embeddings.weight"]
            if cfg.prefix_mode == 0:  # valle.py:1104-1108
                y_emb[:, :Tp] += emb[prompts[..., i + 1]]
            y_emb[:, Tp:] += emb[samples]
    return out


def continual(sd, cfg: OracleConfig, x, x_lens, y) -> torch.Tensor:
    """valle.py:1139-1238 -- NAR-only continuation of given first-codebook codes."""
    assert y.shape[0] == 1 and cfg.num_quantizers == 8
    text_len = int(x_lens.max())
    Tp = min(int(y.shape[1] * 0.5), 3 * 75)
    prompts = y[:, :Tp]
    codes = [y[:, Tp:, 0]]
    # NOTE valle.py:1193-1194 applies position before prenet in the prefix_mode==0 branch;
    # with add_prenet=False (Identity) the two orders are identical.
    codes += nar_decode(sd, cfg, x, text_len, y[..., 0], prompts, Tp, trim_text=False)
    return torch.stack(codes, dim=-1)


# --------------------------------------------------------------------------
# KV-cached greedy AR (the algorithm the engine implements), for the
# "KV cache == full recompute" equivalence check.  Valid because text rows only
# attend to text and audio rows to text + causal audio (valle.py:1019-1030).
# --------------------------------------------------------------------------
def ar_decode_kv(sd, cfg: OracleConfig, x, x_lens, y, max_new_tokens=None,
                 collect_logits: bool = False):
    S = int(x_lens.max())
    d, H = cfg.d_model, cfg.nhead
    hd = d // H
    Tp = y.shape[1]
    xe = pos_embed(sd["ar_text_embedding.word_embeddings.weight"][x[0]],
                   sd["ar_text_position.alpha"])              # [S,d]
    ye = pos_embed(sd["ar_audio_embedding.word_embeddings.weight"][y[0, :, 0]],
                   sd["ar_audio_position.alpha"])             # [Tp,d]
    pe = sine_pe(Tp + 16 * S + 8, d)
    Kc = [torch.zeros(H, 0, hd) for _ in range(cfg.num_layers)]
    Vc = [torch.zeros(H, 0, hd) for _ in range(cfg.num_layers)]

    def run(rows: torch.Tensor, kv_len_of_row) -> torch.Tensor:
        """rows [M,d] appended at the end of the cache; row m sees cache[:kv_len_of_row(m)]."""
        h = rows
        M = rows.shape[0]
        for i in range(cfg.num_layers):
            p = _layer_keys("ar_decoder", i)
            n = layer_norm(h, sd[p + "norm1.weight"], sd[p + "norm1.bias"])
            qkv = F.linear(n, sd[p + "self_attn.in_proj_weight"], sd[p + "self_attn.in_proj_bias"])
            q = qkv[:, :d].view(M, H, hd).transpose(0, 1)
            k = qkv[:, d:2 * d].view(M, H, hd).transpose(0, 1)
            v = qkv[:, 2 * d:].view(M, H, hd).transpose(0, 1)
            Kc[i] = torch.cat([Kc[i], k], dim=1)
            Vc[i] = torch.cat([Vc[i], v], dim=1)
            s = torch.matmul(q, Kc[i].transpose(-1, -2)) * (1.0 / math.sqrt(hd))  # [H,M,Ltot]
            Ltot = Kc[i].shape[1]
            lens = torch.tensor([kv_len_of_row(m) for m in range(M)])
            blocked = torch.arange(Ltot)[None, :] >= lens[:, None]
            s = s.masked_fill(blocked[None], float("-inf"))
            o = torch.matmul(torch.softmax(s, dim=-1), Vc[i]).transpose(0, 1).reshape(M, d)
            h = h + F.linear(o, sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"])
            n = layer_norm(h, sd[p + "norm2.weight"], sd[p + "norm2.bias"])
            h = h + F.linear(F.relu(F.linear(n, sd[p + "linear1.weight"], sd[p + "linear1.bias"])),
                             sd[p + "linear2.weight"], sd[p + "linear2.bias"])
        return layer_norm(h, sd["ar_decoder.norm.weight"], sd["ar_decoder.norm.bias"])

    # prefill: text rows see S keys; audio prompt row j (global S+j) sees S+j+1 keys
    pre = torch.cat([xe, ye], dim=0)
    dec = run(pre, lambda m: S if m < S else m + 1)
    toks: List[int] = []
    logits_all = []
    last = dec[-1:]
    while True:
        logits = F.linear(last, sd["ar_predict_layer.weight"])
        if collect_logits:
            logits_all.append(logits[0].clone())
        tok = int(torch.argmax(logits, dim=-1)[0])
        n_new = len(toks)
        if (tok == NUM_AUDIO_TOKENS or n_new > 16 * S
                or (max_new_tokens is not None and n_new >= max_new_tokens)):
            if n_new == 0:
                raise SyntaxError("well trained model shouldn't reach here.")
            break
        toks.append(tok)
        pos = Tp + n_new
        row = sd["ar_audio_embedding.word_embeddings.weight"][tok][None] \
            + sd["ar_audio_position.alpha"] * pe[pos][None]
        total = S + pos + 1
        last = run(row, lambda m: total)
    out = torch.tensor(toks, dtype=torch.int64)[None]
    return (out, logits_all) if collect_logits else out


# --------------------------------------------------------------------------
# VALLE.forward (training loss) -- restated for the "training forward" row
# --------------------------------------------------------------------------
def weight_checksums(sd) -> Dict[str, torch.Tensor]:
    """Order-independent exact fingerprint of every tensor: int64 sums over the raw fp32 bit
    patterns (plain and position-weighted).  Integer arithmetic, so it does not depend on the
    host's vector width -- a float64 sum does."""
    out = {}
    for k, v in sd.items():
        bits = v.detach().cpu().contiguous().view(-1).view(torch.int32).to(torch.int64)
        w = (torch.arange(bits.numel(), dtype=torch.int64) % 251) + 1
        out[k] = torch.stack([bits.sum(), (bits * w).sum()])
    return out


def make_pad_mask(lengths: torch.Tensor, max_len: int = 0) -> torch.Tensor:
    """icefall.utils.make_pad_mask as called at valle.py:804-805."""
    max_len = max(max_len, int(lengths.max()))
    return torch.arange(max_len)[None, :] >= lengths[:, None]


def forward_train(sd, cfg: OracleConfig, x, x_lens, y, y_lens, nar_stage: int,
                  prefix_len: int, train_stage: int = 0, reduction: str = "sum"):
    """valle.py:762-959 for prefix_mode in {0,1}; `nar_stage` (valle.py:891-895) and
    `prefix_len` (valle.py:348-350, torch.randint) are passed in by the caller so that the
    restatement is deterministic.  Returns (loss, {"ar_logits","nar_logits"})."""
    assert cfg.prefix_mode in (0, 1)
    N, H = x.shape[0], cfg.nhead
    x_mask = make_pad_mask(x_lens)
    y_mask = make_pad_mask(y_lens)
    y_mask_int = y_mask.long()
    codes = y.long() * (1 - y_mask_int.unsqueeze(-1))
    # pad_y_eos valle.py:322-333 (prepend_bos False)
    tg = F.pad(codes[..., 0], (0, 1), value=0) + NUM_AUDIO_TOKENS * F.pad(y_mask_int, (0, 1), value=1)
    yin, targets = tg[:, :-1], tg[:, 1:]
    x_len = int(x_lens.max())
    y_len = int(y_lens.max())
    total = torch.zeros(())
    aux = {}
    if train_stage in (0, 1):
        xe = pos_embed(sd["ar_text_embedding.word_embeddings.weight"][x], sd["ar_text_position.alpha"])
        blocked = ar_inference_mask(x_len, y_len)                       # valle.py:835-848
        pad = torch.concat([x_mask, y_mask], dim=1)                      # valle.py:820
        blocked = blocked[None].logical_or(pad[:, None, :])              # valle.py:852-857
        ye = pos_embed(sd["ar_audio_embedding.word_embeddings.weight"][yin], sd["ar_audio_position.alpha"])
        xy = torch.concat([xe, ye], dim=1)
        fmask = torch.zeros(blocked.shape).masked_fill(blocked, float("-inf"))
        fmask = fmask[:, None].expand(-1, H, -1, -1).reshape(N * H, x_len + y_len, x_len + y_len)
        dec = encoder(sd, "ar_decoder", xy, cfg, blocked=fmask)
        logits = F.linear(dec[:, x_len:], sd["ar_predict_layer.weight"]).permute(0, 2, 1)
        total = total + F.cross_entropy(logits, targets, reduction=reduction)
        aux["ar_logits"] = logits
    if cfg.num_quantizers > 1 and train_stage in (0, 2):
        xe = pos_embed(sd["nar_text_embedding.word_embeddings.weight"][x], sd["nar_text_position.alpha"])
        yq = codes[..., 0]
        if cfg.prefix_mode == 0:                                         # valle.py:339-345
            prefix_len = 0
            y_emb = sd["nar_audio_embeddings.0.word_embeddings.weight"][yq]
            for j in range(1, nar_stage):
                y_emb = y_emb + sd[f"nar_audio_embeddings.{j}.word_embeddings.weight"][codes[..., j]]
        else:                                                            # valle.py:346-362
            y_prompts = sd["nar_audio_embeddings.0.word_embeddings.weight"][yq[:, :prefix_len]].clone()
            y_emb = sd["nar_audio_embeddings.0.word_embeddings.weight"][yq[:, prefix_len:]].clone()
            for j in range(1, cfg.num_quantizers):
                w = sd[f"nar_audio_embeddings.{j}.word_embeddings.weight"]
                y_prompts += w[codes[:, :prefix_len, j]]
                if j < nar_stage:
                    y_emb += w[codes[:, prefix_len:, j]]
            y_emb = torch.concat([y_prompts, y_emb], dim=1)
        tgt = codes[..., nar_stage] + NUM_AUDIO_TOKENS * y_mask_int
        if cfg.prefix_mode == 1:
            tgt = tgt[:, prefix_len:]
        xy = torch.concat([xe, pos_embed(y_emb, sd["nar_audio_position.alpha"])], dim=1)
        pad = torch.concat([x_mask, y_mask], dim=1)
        dec = encoder(sd, "nar_decoder", xy, cfg, key_padding=pad,
                      stage_emb=sd[f"nar_stage_embeddings.{nar_stage - 1}.word_embeddings.weight"])
        dec = dec[:, x_len + prefix_len:]
        logits = F.linear(dec, sd[f"nar_predict_layers.{nar_stage - 1}.weight"]).permute(0, 2, 1)
        tl = y_lens.sum().float()
        total = total + F.cross_entropy(logits, tgt, ignore_index=NUM_AUDIO_TOKENS,
                                        reduction=reduction) * (tl / (tl - prefix_len * N))
        aux["nar_logits"] = logits
    if train_stage == 0:
        total = total / 2.0
    return total, aux
