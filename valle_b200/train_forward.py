"""VALLE.forward (training loss, valle/models/valle.py:762-959) on the sm_90a kernels.

Embeddings + sine PE, the AR stack over padded [text | audio] rows with the merged causal / key-padding rule, one
NAR stage with AdaLN, the prediction heads (tensor-core GEMMs in bf16 mode), cross-entropy and top-10 accuracy.
With gradients enabled (bin/trainer.py:525-531,674: `loss = model(...)`, `scaler.scale(loss).backward()`) every step
goes through the autograd bridges of valle_b200/autograd.py, whose backward runs the gradient kernels of
csrc/backward.cu; under torch.no_grad() (validation) the same kernels run without recording.  In training mode
(`model.train()`) the reference's Dropout sites are live: stateless hashed masks inside the kernels (DESIGN.md).
"""
from __future__ import annotations

from typing import Dict, Tuple, Union

import torch
import torch.nn.functional as F

from . import _lib as L
from . import ops
from .models.macros import NUM_AUDIO_TOKENS


def _make_pad_mask(lengths: torch.Tensor, max_len: int = 0) -> torch.Tensor:
    """icefall.utils.make_pad_mask as called at valle.py:804-805."""
    max_len = max(max_len, int(lengths.max()))
    return torch.arange(max_len, device=lengths.device)[None, :] >= lengths[:, None]


def _top10(logits: torch.Tensor, targets: torch.Tensor, ignore: int) -> torch.Tensor:
    """MulticlassAccuracy(top_k=10, average="micro", ignore_index=ignore) (valle.py:157-163)."""
    keep = targets != ignore
    hit = (logits.topk(10, dim=-1).indices == targets[:, None]).any(-1) & keep
    return hit.sum().float() / keep.sum().clamp(min=1).float()


def valle_forward(model, x: torch.Tensor, x_lens: torch.Tensor, y, y_lens, reduction: str = "sum",
                  train_stage: int = 0, **kwargs):
    """dispatch: with autograd recording if gradients are enabled and any parameter wants one, else forward only"""
    want_grad = torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters())
    if want_grad:
        return _valle_forward(model, x, x_lens, y, y_lens, reduction, train_stage, True, **kwargs)
    with torch.no_grad():
        return _valle_forward(model, x, x_lens, y, y_lens, reduction, train_stage, False, **kwargs)


def _valle_forward(model, x: torch.Tensor, x_lens: torch.Tensor, y, y_lens, reduction: str, train_stage: int,
                   want_grad: bool, **kwargs):
    """VALLE.forward of valle/models/valle.py:762-959 without the backward pass: AR stage (:807-877, causal mask
    of :835-861 as VB_MASK_PADDED_AR), one random NAR stage (:879-941, prefix modes of _prepare_prompts :335-393),
    cross-entropy with reduction `sum` (:877, :936-941) and the top-10 accuracies; returns ((x, codes), loss, metrics)."""
    from . import autograd as AG
    from .models.valle import PromptedFeatures
    assert x.ndim == 2, x.shape
    assert x_lens.ndim == 1, x_lens.shape
    y_prompts_codes = None
    if isinstance(y, PromptedFeatures):
        y_prompts_codes, y = y.data
        prompts_len, y_lens = y_lens.data
        assert prompts_len.min() == prompts_len.max()
        assert model.prefix_mode == 4
        y_prompts_codes = y_prompts_codes.type(torch.int64)
    assert y.ndim == 3, y.shape
    assert y_lens.ndim == 1, y_lens.shape
    assert reduction == "sum", "only reduction='sum' (the trainer's setting) is built"
    dev = model.ar_predict_layer.weight.device
    if dev.type != "cuda":
        raise L.VbError("valle_b200: the model must live on a CUDA device (no CPU fallback)")
    dtype = model.engine_dtype
    if torch.is_autocast_enabled():
        # bin/trainer.py:525 wraps the call in torch.cuda.amp.autocast(dtype=...): reduced-precision autocast selects
        # the tensor-core (bf16 storage, fp32 accumulate) path; fp16 autocast is served by the same bf16 kernels
        try:
            ac = torch.get_autocast_dtype("cuda")
        except Exception:
            ac = torch.get_autocast_gpu_dtype()
        if ac in (torch.bfloat16, torch.float16):
            dtype = torch.bfloat16
    x, y = x.to(dev), y.to(dev)
    x_lens, y_lens = x_lens.to(dev), y_lens.to(dev)
    N, d, Q = x.shape[0], model.ar_predict_layer.weight.shape[1], model.num_quantizers
    x_mask = _make_pad_mask(x_lens)
    y_mask = _make_pad_mask(y_lens)
    y_mask_int = y_mask.type(torch.int64)
    text = x.to(torch.int64).contiguous()
    codes = (y.type(torch.int64) * (1 - y_mask_int.unsqueeze(dim=-1))).contiguous()
    yin, targets = model.pad_y_eos(codes[..., 0], y_mask_int, eos_id=NUM_AUDIO_TOKENS)
    Smax, Tmax = int(x_lens.max()), int(y_lens.max())
    xl32, yl32 = x_lens.to(torch.int32).contiguous(), y_lens.to(torch.int32).contiguous()
    metrics: Dict[str, torch.Tensor] = {}
    total_loss = torch.zeros((), device=dev)
    x_emb_out = None
    eng = None
    # valle.py:830,864,898,918: pre-nets between embedding and position.  Evaluation without gradients runs the engine's
    # folded pre-nets (BatchNorm1d on its running statistics folded into the conv weights, Dropout = identity); training
    # mode or gradients run them through autograd.TextPrenet / AudioPrenet (batch statistics in train(), which update
    # the running statistics in place even under torch.no_grad(), as nn.BatchNorm1d does)
    prenet = getattr(model, "add_prenet", False)
    native_prenet = prenet and (want_grad or model.training)
    if prenet and not native_prenet:
        eng = model.engine()
        eng._refresh()

    def text_prenet(e, name, T):
        if eng is not None:
            # the reference convolves the padded batch: pad-token embeddings inside, zeros beyond the longest text
            return eng._text_prenet(e, [T] * N, name)
        seq = getattr(model, name + "_prenet")
        return AG.TextPrenet.apply(e, seq, T, dtype, drop_seed, AG.PRENET_SITES[name], *AG.text_prenet_params(seq))

    def audio_prenet(rows, name):
        if eng is not None:
            return eng._audio_prenet(rows, name)
        seq = getattr(model, name + "_prenet")
        return AG.AudioPrenet.apply(rows, seq, dtype, drop_seed, AG.PRENET_SITES[name], *AG.audio_prenet_params(seq))

    def embed_pe(tokens, table, pos_mod, T, prenet_name=None, site=None):
        """[N, T] ids -> [N, T, d] = dropout(prenet(table[ids]) + alpha * pe[:T]); prenet_name: "ar_text" / "nar_text"
        (the text pre-nets), "ar_audio" (the AR audio pre-net unless `table` already holds it) or None"""
        tok = tokens.reshape(-1).contiguous()
        e = AG.EmbedSum.apply(tok, 1, 0, tok.numel(), table)
        if prenet and prenet_name in ("ar_text", "nar_text"):
            e = text_prenet(e, prenet_name, T)
        elif native_prenet and prenet_name == "ar_audio":
            e = audio_prenet(e, prenet_name)
        return add_pe(e.view(N, T, table.shape[1]), pos_mod, T, site)

    # training mode (model.train(), bin/trainer.py:512): the Dropout modules of the reference are live -- after every
    # positional encoding (embedding.py:97; p = 0.1, nar_text 0.0) and inside the layers (attention probabilities,
    # both sub-layer outputs, FFN hidden; transformer.py:315-334, p = 0.1).  One seed per call from the device's
    # generator, which is the one the reference's dropout kernels consume (torch.manual_seed reproduces a step, the CPU
    # stream of prefix_len / nar_stage stays aligned with the reference); the masks are the library's stateless hash.
    drop_seed = int(torch.randint(0, 2 ** 62, (1,), device=dev).item()) if model.training else 0
    pe_sites = {"ar_text": 1, "ar_audio": 2, "nar_text": 3, "nar_audio": 4}

    def add_pe(e, pos_mod, T, site=None):
        out = AG.AddPe.apply(e, pos_mod.table(T, dev), pos_mod.alpha)
        if model.training and site is not None and pos_mod.dropout.p > 0:
            out = AG.Dropout.apply(out, pos_mod.dropout.p, drop_seed, 0x10000 + pe_sites[site])
        return out

    def stack(enc, nd, rows, seg1_lens, mode, ada=None, Lp=None, seed_offset=0):
        cu = (torch.arange(N + 1, dtype=torch.int32, device=dev) * Lp).contiguous()
        p_layer = float(enc.layers[0].dropout.p) if model.training else 0.0
        if want_grad or p_layer > 0:
            return AG.DecoderStack.apply(rows, ada, nd, (cu, N, Lp, mode, xl32, seg1_lens, Smax, p_layer,
                                                         drop_seed + seed_offset), *AG.layer_params(enc))
        nd.forward(rows, cu, N, Lp, mode, xl32, ada, seg1_lens=seg1_lens, seg1_start=Smax)
        return rows

    def final_norm(nd, rows, ada, sel):
        fn = nd.enc.norm
        if fn is None:   # post-LN stacks have no final norm (valle.py:151,242-246)
            return AG.GatherRows.apply(rows, sel, dtype)
        wb = ada[2 * nd.n_layer] if ada is not None else None
        inner = fn.norm if ada is not None else fn
        return AG.LayerNormRows.apply(rows, inner.weight, inner.bias, wb, sel, inner.eps, dtype)

    def ada_table(enc, nd, stage_weight):
        if not want_grad:
            return nd.ada_table(stage_weight)
        wb = []
        for lyr in enc.layers:
            for nm in (lyr.norm1, lyr.norm2):
                wb += [nm.project_layer.weight, nm.project_layer.bias]
        if enc.norm is not None:
            wb += [enc.norm.project_layer.weight, enc.norm.project_layer.bias]
        return AG.AdaTable.apply(stage_weight, *wb)

    # ---- AR decoder (valle.py:828-881) ----
    if train_stage in (0, 1):
        xe = embed_pe(text, model.ar_text_embedding.weight, model.ar_text_position, Smax, "ar_text", "ar_text")
        Ta = yin.shape[1]                     # Tmax, or Tmax + 1 with the prepended <BOS> (valle.py:820-826,833)
        ar_table = eng.ar_audio_table if eng is not None else model.ar_audio_embedding.weight   # pre-net(embedding)
        ye = embed_pe(yin.contiguous(), ar_table, model.ar_audio_position, Ta, "ar_audio", "ar_audio")
        rows = torch.cat([xe, ye], dim=1).reshape(N * (Smax + Ta), d).contiguous()
        nd = model.ar_decoder.native(dtype)
        yl_ar = (yl32 + (Ta - Tmax)).contiguous()
        rows = stack(model.ar_decoder, nd, rows, yl_ar, L.VB_MASK_PADDED_AR, None, Smax + Ta)
        sel = (torch.arange(N, device=dev)[:, None] * (Smax + Ta) + Smax
               + torch.arange(Ta, device=dev)[None, :]).reshape(-1).to(torch.int32).contiguous()
        hn = final_norm(nd, rows, None, sel)
        logits = AG.Linear.apply(hn, model.ar_predict_layer.weight, dtype)
        tg = targets.reshape(-1).contiguous()
        total_loss = total_loss + AG.CrossEntropySum.apply(logits, tg, -1)
        metrics["ArTop10Accuracy"] = _top10(logits.detach(), tg, NUM_AUDIO_TOKENS).item() * y_lens.sum().type(torch.float32)
        x_emb_out = xe

    if Q == 1:
        return ((x_emb_out, codes), total_loss, metrics)

    # ---- NAR decoder, one random stage (valle.py:886-954) ----
    if train_stage in (0, 2):
        num_nar_layers = Q - 1
        nar_stage = model.rng.choices([_k for _k in range(1, Q)], weights=[1.0 / num_nar_layers] * num_nar_layers, k=1)[0]
        xe = embed_pe(text, model.nar_text_embedding.weight, model.nar_text_position, Smax, "nar_text", "nar_text")
        emb = [e.weight for e in model.nar_audio_embeddings]
        yq = codes[..., 0].contiguous()
        pm = model.prefix_mode

        def emb_sum(tok2d, tabs, T):  # [N, T, len(tabs)] ids -> sum_j tabs[j][ids[..., j]] in order
            tok = tok2d.reshape(-1, len(tabs)).contiguous()
            return AG.EmbedSum.apply(tok, len(tabs), 1, tok.shape[0], *tabs).view(N, T, tabs[0].shape[1])

        if pm == 0:  # valle.py:339-345
            prefix_len = 0
            y_emb = emb_sum(codes[..., :nar_stage], emb[:nar_stage], Tmax)
        elif pm == 1:  # valle.py:346-362
            int_low = (0.25 * y_lens.min()).type(torch.int64).item()
            prefix_len = torch.randint(int_low, int_low * 2, size=()).item()
            prefix_len = min(prefix_len, 225)
            y_prompts = emb_sum(codes[:, :prefix_len], emb[:Q], prefix_len)
            y_rest = emb_sum(codes[:, prefix_len:, :nar_stage], emb[:nar_stage], Tmax - prefix_len)
            y_emb = torch.cat([y_prompts, y_rest], dim=1)
        elif pm in (2, 4):  # valle.py:363-389
            if pm == 2:
                prefix_len = min(225, int(0.25 * y_lens.min().item()))
                pcs = []
                for b in range(N):
                    start = model.rng.randint(0, y_lens[b].item() - prefix_len)
                    pcs.append(torch.clone(codes[b, start:start + prefix_len]))
                    codes[b, start:start + prefix_len, nar_stage] = NUM_AUDIO_TOKENS
                y_prompts_codes = torch.stack(pcs, dim=0)
            else:
                prefix_len = y_prompts_codes.shape[1]
                y_prompts_codes = y_prompts_codes.to(dev)
            y_prompts = emb_sum(y_prompts_codes, emb[:Q], prefix_len)
            y_rest = emb_sum(codes[..., :nar_stage], emb[:nar_stage], Tmax)
            y_emb = torch.cat([y_prompts, y_rest], dim=1)
        else:
            raise ValueError
        tg = codes[..., nar_stage] + NUM_AUDIO_TOKENS * y_mask_int
        Ty = y_emb.shape[1]
        seg1 = yl32
        if pm in (2, 4):
            seg1 = (yl32 + (Ty - Tmax)).contiguous()   # key mask F.pad(y_mask, (prefix, 0), False) valle.py:908-914
        elif pm == 1:
            tg = tg[:, prefix_len:]
        if prenet:   # valle.py:918
            y_emb = audio_prenet(y_emb.reshape(N * Ty, -1).contiguous(), "nar_audio").view(N, Ty, -1)
        y_pos = add_pe(y_emb.contiguous(), model.nar_audio_position, Ty, "nar_audio")
        Lp = Smax + Ty
        rows = torch.cat([xe, y_pos], dim=1).reshape(N * Lp, xe.shape[-1]).contiguous()
        nd = model.nar_decoder.native(dtype)
        ada = ada_table(model.nar_decoder, nd, model.nar_stage_embeddings[nar_stage - 1].weight)
        rows = stack(model.nar_decoder, nd, rows, seg1, L.VB_MASK_PADDED, ada, Lp, seed_offset=1)
        off = Smax + prefix_len
        if pm == 4:
            off = Smax + prefix_len
        Tt = Lp - off
        sel = (torch.arange(N, device=dev)[:, None] * Lp + off
               + torch.arange(Tt, device=dev)[None, :]).reshape(-1).to(torch.int32).contiguous()
        hn = final_norm(nd, rows, ada, sel)
        logits = AG.Linear.apply(hn, model.nar_predict_layers[nar_stage - 1].weight, dtype)
        tgf = tg.reshape(-1).contiguous()
        if pm == 4:
            prefix_len = 0  # reset for the metric / loss rescale (valle.py:927-928)
        total_length = y_lens.sum().type(torch.float32)
        ce = AG.CrossEntropySum.apply(logits, tgf, NUM_AUDIO_TOKENS)
        total_loss = total_loss + ce * (total_length / (total_length - prefix_len * N))
        lp = F.pad(logits.detach(), (0, 1), value=logits.min().item())   # valle.py:946-950
        metrics["NarTop10Accuracy"] = _top10(lp, tgf, NUM_AUDIO_TOKENS).item() * total_length
        x_emb_out = xe
    if train_stage == 0:
        total_loss = total_loss / 2.0
    return ((x_emb_out, codes), total_loss, metrics)
