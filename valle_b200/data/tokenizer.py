"""AudioTokenizer with the reference's interface (valle/data/tokenizer.py:211-254): EnCodec 24 kHz at
6 kbps (8 codebooks of 1024), `.encode(wav) -> [(codes [B, 8, T'], None)]`, `.decode(frames) -> wav`,
`.sample_rate`, `.channels`, `.device` -- running on the sm_90a kernels of libvalle_b200.so
(`csrc/encodec.cu`: SConv1d / SConvTranspose1d with reflect padding and ELU pre-activation, the
2-layer LSTM, the 8-stage residual VQ; `vb_linear` for the LSTM input projections, `vb_embed_sum`
for the RVQ decode).

The reference gets the weights from `EncodecModel.encodec_model_24khz()` (PyPI `encodec`, downloaded at
run time) and strips weight-norm (`remove_encodec_weight_norm`, tokenizer.py:181-208).  Neither the package
nor the weights exist offline, so this class takes a state dict in the layout of
`transformers.EncodecModel` ("facebook/encodec_24khz": `encoder.layers.N.conv.*`, `…lstm.*`,
`quantizer.layers.Q.codebook.embed`), with or without the weight-norm parametrisation, and folds it at
load.  No CPU fallback.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from .. import _lib as L
from .. import ops


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class _Conv:
    """one SConv1d: folded weight [Cout, Cin, K], bias, stride, dilation."""

    def __init__(self, w: torch.Tensor, b: torch.Tensor, stride: int = 1, dilation: int = 1):
        self.b, self.stride, self.dilation = b.contiguous(), stride, dilation
        self.cout, self.cin, self.k = w.shape
        self.wp = w.permute(1, 2, 0).contiguous()   # [Cin, K, Cout]: the layout the tiled kernel streams

    def __call__(self, x: torch.Tensor, pre_elu: bool = False, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        B, Cin, Tin = x.shape
        assert Cin == self.cin
        eff_k = (self.k - 1) * self.dilation + 1
        padding_total = eff_k - self.stride
        # extra right padding so the last window is complete (encodec `pad_for_conv1d`)
        n_frames = math.ceil((Tin - eff_k + padding_total) / self.stride + 1) - 1
        extra = n_frames * self.stride + eff_k - padding_total - Tin
        Tout = (Tin + padding_total + extra - eff_k) // self.stride + 1
        out = torch.empty((B, self.cout, Tout), dtype=torch.float32, device=x.device)
        L.check(L.load().vb_conv1d(x.data_ptr(), B, Cin, Tin, self.wp.data_ptr(), self.b.data_ptr(), self.cout, self.k,
                                   self.stride, self.dilation, padding_total, extra, 1, int(pre_elu), L.ptr(residual),
                                   out.data_ptr(), Tout, 1, _stream()), "vb_conv1d")
        return out


class _ConvT:
    """causal SConvTranspose1d (K = 2 * stride, right padding trimmed) as a stride-1 two-tap convolution onto
    Cout * stride phase channels: out[co, q*s + r] = sum_ci x[ci, q] w[ci, co, r] + x[ci, q-1] w[ci, co, r + s]"""

    def __init__(self, w: torch.Tensor, b: torch.Tensor, stride: int):
        self.b, self.stride = b.contiguous(), stride
        self.cin, self.cout, self.k = w.shape
        assert self.k == 2 * stride, "EnCodec up-sampling layers have K == 2 * stride"
        s = stride
        wp = torch.empty((self.cin, 2, self.cout * s), dtype=w.dtype, device=w.device)
        wp[:, 0] = w[:, :, s:].reshape(self.cin, self.cout * s)   # tap 0 multiplies x[q - 1]
        wp[:, 1] = w[:, :, :s].reshape(self.cin, self.cout * s)   # tap 1 multiplies x[q]
        self.wp = wp.contiguous()

    def __call__(self, x: torch.Tensor, pre_elu: bool = False) -> torch.Tensor:
        B, Cin, Tin = x.shape
        s = self.stride
        out = torch.empty((B, self.cout, Tin * s), dtype=torch.float32, device=x.device)
        L.check(L.load().vb_conv1d(x.data_ptr(), B, Cin, Tin, self.wp.data_ptr(), self.b.data_ptr(), self.cout * s, 2,
                                   1, 1, 1, 0, 0, int(pre_elu), 0, out.data_ptr(), Tin, s, _stream()), "vb_conv1d")
        return out


class _Res:
    """SEANetResnetBlock: shortcut_1x1(x) + conv_k1(ELU(conv_k3(ELU(x))))."""

    def __init__(self, c1: _Conv, c2: _Conv, sc: _Conv):
        self.c1, self.c2, self.sc = c1, c2, sc

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        s = self.sc(x)
        return self.c2(self.c1(x, pre_elu=True), pre_elu=True, residual=s)


class _LSTM:
    def __init__(self, layers: List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]):
        self.layers = layers  # (W_ih [4H, In], bias_ih + bias_hh [4H], W_hh^T [H, 4H])

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """x [B, C, T] -> LSTM(x) + x (skip), same layout."""
        B, Cc, T = x.shape
        lib = L.load()
        seq = torch.empty((T, B, Cc), dtype=torch.float32, device=x.device)
        L.check(lib.vb_permute3(x.data_ptr(), B, Cc, T, 2, 0, 1, seq.data_ptr(), _stream()), "vb_permute3")
        inp = seq
        for w_ih, bias, whh_t in self.layers:
            H = whh_t.shape[0]
            xproj = ops.linear(inp.view(T * B, -1), w_ih, bias)          # [T*B, 4H]
            h_seq = torch.empty((T, B, H), dtype=torch.float32, device=x.device)
            c = torch.empty(B * H + 64, dtype=torch.float32, device=x.device)
            L.check(lib.vb_lstm_layer(xproj.data_ptr(), whh_t.data_ptr(), T, B, H, h_seq.data_ptr(), c.data_ptr(),
                                      _stream()), "vb_lstm_layer")
            inp = h_seq
        out = torch.empty_like(x)
        # skip connection of EncodecLSTM / SLSTM: y = lstm(x) + x, as out = in + 1.0 * table rows
        y = torch.empty((T * B, Cc), dtype=torch.float32, device=x.device)
        ops.add_pe(inp.view(T * B, Cc), seq.view(T * B, Cc), self.one(x.device), y, T * B, pos0=0)
        L.check(lib.vb_permute3(y.data_ptr(), T, B, Cc, 1, 2, 0, out.data_ptr(), _stream()), "vb_permute3")
        return out

    _ones = {}

    @classmethod
    def one(cls, device):
        if device not in cls._ones:
            cls._ones[device] = torch.ones(1, dtype=torch.float32, device=device)
        return cls._ones[device]


def _fold(sd: Dict[str, torch.Tensor], prefix: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """effective conv weight: plain `weight`, or weight-norm g * v / ||v|| over dims (1, 2)."""
    if prefix + ".weight" in sd:
        w = sd[prefix + ".weight"]
    else:
        g = sd[prefix + ".parametrizations.weight.original0"] if prefix + ".parametrizations.weight.original0" in sd \
            else sd[prefix + ".weight_g"]
        v = sd[prefix + ".parametrizations.weight.original1"] if prefix + ".parametrizations.weight.original1" in sd \
            else sd[prefix + ".weight_v"]
        w = v * (g / v.norm(2, dim=(1, 2), keepdim=True))
    return w.float(), sd[prefix + ".bias"].float()


def random_encodec_weights(seed: int = 0, n_q: int = 8) -> Dict[str, torch.Tensor]:
    """A state dict of the published EnCodec 24 kHz architecture (transformers.EncodecModel key names, plain
    `.conv.weight` form) with seeded random values: ratios 8*5*4*2, 32 base filters, residual blocks with a k=3 /
    k=1 pair and a 1x1 shortcut, 2-layer LSTM of 512, 128-dim latents, 1024 x 128 codebooks.  For synthetic
    benchmarks and smoke tests when no trained weights are at hand (the reference downloads them)."""
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def conv(prefix, cout, cin, k):
        bound = 1.0 / math.sqrt(cin * k)
        sd[prefix + ".conv.weight"] = (torch.rand(cout, cin, k, generator=g) * 2 - 1) * bound
        sd[prefix + ".conv.bias"] = (torch.rand(cout, generator=g) * 2 - 1) * bound

    def convt(prefix, cin, cout, k):
        bound = 1.0 / math.sqrt(cin * k)
        sd[prefix + ".conv.weight"] = (torch.rand(cin, cout, k, generator=g) * 2 - 1) * bound
        sd[prefix + ".conv.bias"] = (torch.rand(cout, generator=g) * 2 - 1) * bound

    def res(prefix, ch):
        conv(prefix + ".block.1", ch // 2, ch, 3)
        conv(prefix + ".block.3", ch, ch // 2, 1)
        conv(prefix + ".shortcut", ch, ch, 1)

    def lstm(prefix, h):
        b = 1.0 / math.sqrt(h)
        for i in range(2):
            for nm, shp in (("weight_ih", (4 * h, h)), ("weight_hh", (4 * h, h)), ("bias_ih", (4 * h,)), ("bias_hh", (4 * h,))):
                sd[f"{prefix}.lstm.{nm}_l{i}"] = (torch.rand(*shp, generator=g) * 2 - 1) * b

    ratios = EncodecNative.RATIOS
    ch = 32
    conv("encoder.layers.0", ch, 1, 7)
    i = 1
    for r in reversed(ratios):
        res(f"encoder.layers.{i}", ch)
        conv(f"encoder.layers.{i + 2}", 2 * ch, ch, 2 * r)
        ch *= 2
        i += 3
    lstm(f"encoder.layers.{i}", ch)
    conv(f"encoder.layers.{i + 2}", 128, ch, 7)
    conv("decoder.layers.0", ch, 128, 7)
    lstm("decoder.layers.1", ch)
    i = 2
    for r in ratios:
        convt(f"decoder.layers.{i + 1}", ch, ch // 2, 2 * r)
        ch //= 2
        res(f"decoder.layers.{i + 2}", ch)
        i += 3
    conv(f"decoder.layers.{i + 1}", 1, ch, 7)
    for q in range(n_q):
        sd[f"quantizer.layers.{q}.codebook.embed"] = torch.randn(1024, 128, generator=g) * (0.8 ** q)
    return sd


class EncodecNative:
    """EnCodec 24 kHz encoder / quantizer / decoder on the native kernels."""

    RATIOS = (8, 5, 4, 2)

    def __init__(self, state_dict: Dict[str, torch.Tensor], device, n_q: int = 8):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise L.VbError("valle_b200.AudioTokenizer needs a CUDA device (no CPU fallback)")
        L.load()
        sd = {k: v.detach().to("cpu") for k, v in state_dict.items()}
        self.device, self.n_q = dev, n_q

        def conv(prefix, stride=1, dilation=1):
            w, b = _fold(sd, prefix + ".conv")
            return _Conv(w.to(dev), b.to(dev), stride, dilation)

        def convt(prefix, stride):
            w, b = _fold(sd, prefix + ".conv")
            return _ConvT(w.to(dev), b.to(dev), stride)

        def res(prefix):
            return _Res(conv(prefix + ".block.1"), conv(prefix + ".block.3"), conv(prefix + ".shortcut"))

        def lstm(prefix):
            layers = []
            i = 0
            while f"{prefix}.lstm.weight_ih_l{i}" in sd:
                w_ih = sd[f"{prefix}.lstm.weight_ih_l{i}"].float().contiguous().to(dev)
                bias = (sd[f"{prefix}.lstm.bias_ih_l{i}"] + sd[f"{prefix}.lstm.bias_hh_l{i}"]).float().contiguous().to(dev)
                whh_t = sd[f"{prefix}.lstm.weight_hh_l{i}"].float().t().contiguous().to(dev)
                layers.append((w_ih, bias, whh_t))
                i += 1
            return _LSTM(layers)

        # encoder (SEANetEncoder): conv7, 4 x [resblock, ELU, strided conv], LSTM, ELU, conv7
        self.enc = [("conv", conv("encoder.layers.0"))]
        i = 1
        for r in reversed(self.RATIOS):
            self.enc.append(("res", res(f"encoder.layers.{i}")))
            self.enc.append(("conv_elu", conv(f"encoder.layers.{i + 2}", stride=r)))
            i += 3
        self.enc.append(("lstm", lstm(f"encoder.layers.{i}")))
        self.enc.append(("conv_elu", conv(f"encoder.layers.{i + 2}")))
        # decoder (SEANetDecoder): conv7, LSTM, 4 x [ELU, convT, resblock], ELU, conv7
        self.dec = [("conv", conv("decoder.layers.0")), ("lstm", lstm("decoder.layers.1"))]
        i = 2
        for r in self.RATIOS:
            self.dec.append(("convt_elu", convt(f"decoder.layers.{i + 1}", r)))
            self.dec.append(("res", res(f"decoder.layers.{i + 2}")))
            i += 3
        self.dec.append(("conv_elu", conv(f"decoder.layers.{i + 1}")))
        # residual vector quantiser
        cbs = [sd[f"quantizer.layers.{q}.codebook.embed"].float() for q in range(n_q)]
        self.cb = torch.stack(cbs).contiguous().to(dev)                      # [n_q, 1024, 128]
        self.cb_t = self.cb.transpose(1, 2).contiguous()                     # [n_q, 128, 1024]
        self.cb_sq = torch.stack([c.pow(2).sum(1) for c in cbs]).contiguous().to(dev)
        self.cb_list = [self.cb[q] for q in range(n_q)]
        self.hop = 1
        for r in self.RATIOS:
            self.hop *= r

    @staticmethod
    def _run(stack, x):
        for kind, m in stack:
            if kind == "conv":
                x = m(x)
            elif kind in ("conv_elu", "convt_elu"):
                x = m(x, pre_elu=True)
            else:
                x = m(x)
        return x

    @torch.no_grad()
    def encode(self, wav: torch.Tensor) -> torch.Tensor:
        """wav [B, 1, N] fp32 -> codes [B, n_q, ceil(N / 320)] int64."""
        x = wav.to(self.device, torch.float32).contiguous()
        emb = self._run(self.enc, x)                                      # [B, 128, T']
        B, D, T = emb.shape
        rows = torch.empty((B, T, D), dtype=torch.float32, device=self.device)
        lib = L.load()
        L.check(lib.vb_permute3(emb.data_ptr(), B, D, T, 0, 2, 1, rows.data_ptr(), _stream()), "vb_permute3")
        codes = torch.empty((B, self.n_q, T), dtype=torch.int64, device=self.device)
        # codes[b, q, t] of the whole batch in one launch: frame stride 1, stage stride T, utterance stride n_q * T
        L.check(lib.vb_rvq_encode(rows.data_ptr(), B * T, D, self.n_q, self.cb.shape[1], self.cb.data_ptr(),
                                  self.cb_t.data_ptr(), self.cb_sq.data_ptr(), codes.data_ptr(), 1, T, T, self.n_q * T,
                                  _stream()), "vb_rvq_encode")
        return codes

    @torch.no_grad()
    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        """codes [B, n_q, T'] -> wav [B, 1, T' * 320]."""
        codes = codes.to(self.device, torch.int64)
        B, Q, T = codes.shape
        tok = codes.permute(0, 2, 1).contiguous().view(B * T, Q)            # [rows, Q]
        D = self.cb.shape[2]
        rows = torch.empty((B * T, D), dtype=torch.float32, device=self.device)
        ops.embed_sum(tok, Q, 1, self.cb_list[:Q], B * T, rows)              # sum of the Q codebook vectors
        emb = torch.empty((B, D, T), dtype=torch.float32, device=self.device)
        L.check(L.load().vb_permute3(rows.data_ptr(), B, T, D, 0, 2, 1, emb.data_ptr(), _stream()), "vb_permute3")
        return self._run(self.dec, emb)


class AudioTokenizer:
    """EnCodec audio (valle/data/tokenizer.py:211-242).  `weights`: state dict (or path to a torch-saved one)
    in transformers' EncodecModel layout."""

    def __init__(self, device=None, weights: Union[None, str, Dict[str, torch.Tensor]] = None) -> None:
        if weights is None:
            raise L.VbError(
                "valle_b200.AudioTokenizer: pass weights=<EnCodec 24 kHz state dict or path> (transformers "
                "EncodecModel layout). The reference downloads them through the PyPI `encodec` package, which "
                "is not available offline.")
        if isinstance(weights, str):
            weights = torch.load(weights, map_location="cpu")
        if not device:
            device = torch.device("cuda:0")
        self._device = torch.device(device)
        self.codec = EncodecNative(weights, self._device, n_q=8)   # 6 kbps = 8 codebooks (tokenizer.py:220)
        self.sample_rate = 24000
        self.channels = 1

    @property
    def device(self):
        return self._device

    def encode(self, wav: torch.Tensor):
        return [(self.codec.encode(wav), None)]

    def decode(self, frames) -> torch.Tensor:
        codes = torch.cat([f[0] for f in frames], dim=-1) if len(frames) > 1 else frames[0][0]
        return self.codec.decode(codes)


def tokenize_audio(tokenizer: AudioTokenizer, wav: torch.Tensor, sr: int = 24000):
    """valle/data/tokenizer.py:245-254 for an already-loaded waveform [C, N] at `sr` (resampling / file
    I/O stay with torchaudio in the caller)."""
    assert sr == tokenizer.sample_rate, "resample to 24 kHz first (encodec.utils.convert_audio in the reference)"
    if wav.dim() == 2:
        wav = wav.mean(0, keepdim=True) if wav.shape[0] != tokenizer.channels else wav
        wav = wav.unsqueeze(0)
    with torch.no_grad():
        return tokenizer.encode(wav.to(tokenizer.device))


# ---------------------------------------------------------------------------------------------------------------
# Dataset-scale tokenisation (valle/data/tokenizer.py:256-361, valle/bin/tokenizer.py:172-214)
# ---------------------------------------------------------------------------------------------------------------
def compute_num_frames(duration: float, frame_shift: float, sampling_rate: int) -> int:
    """lhotse.utils.compute_num_frames as called at tokenizer.py:300-304,349-354 (lhotse is an un-vendored
    dependency): the number of frames is duration / frame_shift rounded half up."""
    from decimal import ROUND_HALF_UP, Decimal
    return int(Decimal(round(duration / frame_shift, ndigits=8)).quantize(0, rounding=ROUND_HALF_UP))


class AudioTokenConfig:
    """tokenizer.py:256-267"""

    def __init__(self, frame_shift: float = 320.0 / 24000, num_quantizers: int = 8):
        self.frame_shift = frame_shift
        self.num_quantizers = num_quantizers

    def to_dict(self):
        return dict(frame_shift=self.frame_shift, num_quantizers=self.num_quantizers)

    @staticmethod
    def from_dict(data):
        return AudioTokenConfig(**data)


class AudioTokenExtractor:
    """tokenizer.py:270-361 (an lhotse FeatureExtractor in the reference; lhotse is not a dependency here, the
    methods lhotse calls -- `extract`, `extract_batch`, `frame_shift`, `feature_dim`, `name`, `config` -- are kept).
    Waveforms must already be 24 kHz mono (the reference resamples with encodec.utils.convert_audio, :284-290)."""
    name = "encodec"
    config_type = AudioTokenConfig

    def __init__(self, config: Optional[AudioTokenConfig] = None, tokenizer: Optional[AudioTokenizer] = None,
                 device=None, weights=None, max_batch: int = 32):
        self.config = config or AudioTokenConfig()
        self.tokenizer = tokenizer or AudioTokenizer(device=device, weights=weights)
        self.max_batch = max_batch

    @property
    def frame_shift(self) -> float:
        return self.config.frame_shift

    def feature_dim(self, sampling_rate: int) -> int:
        return self.config.num_quantizers

    def _check_rate(self, sampling_rate: int):
        if sampling_rate != self.tokenizer.sample_rate:
            raise ValueError(f"valle_b200.AudioTokenExtractor: resample to {self.tokenizer.sample_rate} Hz first")

    def extract(self, samples, sampling_rate: int):
        """[1, N] waveform -> numpy [T, 8] codes (tokenizer.py:278-307)"""
        return self.extract_batch([samples], sampling_rate, None)[0]

    def extract_batch_device(self, samples: Sequence, sampling_rate: int) -> List[torch.Tensor]:
        """codes [T_b, 8] int64 ON THE DEVICE for every waveform: utterances are sorted by length and encoded in
        zero-padded batches of <= max_batch; each result is trimmed to its expected frame count (:345-357)"""
        self._check_rate(sampling_rate)
        dev = self.tokenizer.device
        waves = [torch.as_tensor(w).reshape(-1).to(torch.float32) for w in samples]
        order = sorted(range(len(waves)), key=lambda i: -waves[i].numel())
        out: List[Optional[torch.Tensor]] = [None] * len(waves)
        for b0 in range(0, len(order), self.max_batch):
            ids = order[b0:b0 + self.max_batch]
            n_max = waves[ids[0]].numel()
            batch = torch.zeros((len(ids), 1, n_max), dtype=torch.float32, device=dev)
            for j, i in enumerate(ids):
                batch[j, 0, : waves[i].numel()] = waves[i].to(dev, non_blocking=True)
            codes = self.tokenizer.encode(batch)[0][0]                       # [B, n_q, T]
            for j, i in enumerate(ids):
                n = compute_num_frames(round(waves[i].numel() / sampling_rate, ndigits=12), self.frame_shift, sampling_rate)
                assert abs(-(-waves[i].numel() // self.tokenizer.codec.hop) - n) <= 1
                out[i] = codes[j, :, :n].t()                                 # [T, n_q]
        return out

    def extract_batch(self, samples, sampling_rate: int, lengths=None):
        """list of waveforms -> list of numpy [T_b, 8] (tokenizer.py:326-361)"""
        return [c.cpu().numpy() for c in self.extract_batch_device(samples, sampling_rate)]
