"""The e4m3 rule of compute_type="float8_float16" on the CPU (mirror of faster_whisper_b200/csrc/fp8.cuh), and the encoder
that applies it where the engine does.

Per row: scale s = amax / 448 in float32 (a row whose amax is 0 gets s = 1), code q = e4m3(x / s) with the float32 quotient
rounded to nearest-even onto the e4m3 grid and saturated at +-448.  ``torch.float8_e4m3fn`` does the rounding (ties to even);
it turns values beyond 448 into NaN, so they are clamped first, which is what the device's satfinite conversion does.
"""
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle.whisper_oracle import WhisperOracle

E4M3_MAX = 448.0


def round_e4m3(x: torch.Tensor) -> torch.Tensor:
    """float32 -> torch.float8_e4m3fn: round to nearest even, saturating at +-448."""
    return x.float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def quantize_rows(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """float32 [rows, K] -> (codes as torch.float8_e4m3fn [rows, K], float32 scales [rows])."""
    x = x.float()
    amax = x.abs().amax(dim=-1)
    s = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    return round_e4m3(x / s[..., None]), s


def codes_to_bytes(q: torch.Tensor) -> np.ndarray:
    return q.view(torch.uint8).numpy()


def fp8_linear(q: torch.Tensor, s: torch.Tensor, wq: torch.Tensor, ws: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    """s[r] * ws[n] * sum_k q[r][k] wq[n][k] (+ bias) with the products summed in float64; float32 result."""
    acc = q.double() @ wq.double().T
    out = acc * s.double()[:, None] * ws.double()[None, :]
    if bias is not None:
        out = out + bias.double()
    return out.float()


class FP8EncoderOracle(WhisperOracle):
    """WhisperOracle whose encoder runs the four linear layers of each block as the engine's compute_type="float8_float16" does:
    weights quantised per output channel from their fp16 values (Q, K, V as one fused matrix, row by row), the LayerNorm outputs
    from their float32 values, the attention output and GELU(FFN1) after rounding to fp16, products summed in float64.  The conv
    stem, attention, ln_post and the whole decoder are the float32 oracle's."""

    def __init__(self, dims: dict, weights: Dict[str, np.ndarray], tokens: dict, suppress_ids_begin: Optional[Sequence[int]] = None,
                 num_threads: Optional[int] = None):
        super().__init__(dims, weights, tokens, suppress_ids_begin=suppress_ids_begin, num_threads=num_threads)
        d = self.dims["n_audio_state"]
        self.q8 = {}
        for i in range(self.dims["n_audio_layer"]):
            p = f"encoder.blocks.{i}"
            wqkv = torch.cat([self.w[f"{p}.attn.{n}.weight"] for n in ("query", "key", "value")])
            bqkv = torch.cat([self.w[f"{p}.attn.query.bias"], torch.zeros(d), self.w[f"{p}.attn.value.bias"]])
            for name, wt, b in (("qkv", wqkv, bqkv), ("out", self.w[f"{p}.attn.out.weight"], self.w[f"{p}.attn.out.bias"]),
                                ("fc1", self.w[f"{p}.mlp.0.weight"], self.w[f"{p}.mlp.0.bias"]),
                                ("fc2", self.w[f"{p}.mlp.2.weight"], self.w[f"{p}.mlp.2.bias"])):
                q, s = quantize_rows(wt.half().float())
                self.q8[(i, name)] = (q, s, b)

    def _lin8(self, x: torch.Tensor, i: int, name: str) -> torch.Tensor:
        b, t, k = x.shape
        q, s = quantize_rows(x.reshape(b * t, k))
        wq, ws, bias = self.q8[(i, name)]
        return fp8_linear(q, s, wq, ws, bias).reshape(b, t, -1)

    @torch.no_grad()
    def encode(self, features: np.ndarray) -> torch.Tensor:
        x = torch.from_numpy(np.ascontiguousarray(features)).float()
        if x.ndim == 2:
            x = x[None]
        x = F.gelu(F.conv1d(x, self.w["encoder.conv1.weight"], self.w["encoder.conv1.bias"], padding=1))
        x = F.gelu(F.conv1d(x, self.w["encoder.conv2.weight"], self.w["encoder.conv2.bias"], stride=2, padding=1))
        x = x.permute(0, 2, 1) + self.w["encoder.positional_embedding"][: x.shape[-1]]
        d = self.dims["n_audio_state"]
        for i in range(self.dims["n_audio_layer"]):
            p = f"encoder.blocks.{i}"
            qkv = self._lin8(self._ln(x, p + ".attn_ln"), i, "qkv")
            a, _ = self._mha(qkv[..., :d], qkv[..., d:2 * d], qkv[..., 2 * d:], self.n_audio_head)
            x = x + self._lin8(a.half().float(), i, "out")
            h = F.gelu(self._lin8(self._ln(x, p + ".mlp_ln"), i, "fc1"))
            x = x + self._lin8(h.half().float(), i, "fc2")
        return self._ln(x, "encoder.ln_post")
