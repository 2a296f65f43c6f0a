"""CPU oracle for the faster-whisper hot path: log-mel -> Whisper encoder -> CTranslate2-style decoding.

**TEST INFRASTRUCTURE ONLY.**  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import this file, and only as the checker or the timed
CPU baseline.  The product (``faster_whisper_b200``) never imports it and has no CPU fallback.

What is restated, and from where (paths relative to the reference tree):

* ``mel_filters`` / ``log_mel``      <- ``faster_whisper/feature_extractor.py:24-65`` and ``:198-230``
  (**pinned**: checked bit-for-tolerance against the reference class itself, see
  ``oracle/make_golden.py`` and ``tests/test_oracle.py``).
* ``WhisperOracle.encode`` / decoder  <- the OpenAI Whisper architecture that ``ctranslate2.models.Whisper``
  executes (call sites ``faster_whisper/transcribe.py:209,1400``).  CTranslate2 (``ctranslate2>=4.0,<5``,
  ``requirements.txt:1``) is a pip dependency that is *not* vendored in the reference tree and is not
  installed here, so the network math is cross-checked against ``transformers.WhisperForConditionalGeneration``
  with shared weights (``oracle/check_against_transformers.py``) — a check of our restatement, not of CT2.
* ``WhisperOracle.generate``          <- CTranslate2 4.x ``Whisper.generate`` semantics as consumed at
  ``faster_whisper/transcribe.py:222-236,1446-1459``: logits processors (suppress_tokens, suppress_blank,
  Whisper timestamp rules, repetition penalty, no-repeat-ngram), beam search with 2K candidates /
  patience / length penalty applied at finalisation with EOS excluded from the length (the inverse is
  visible in-tree at ``transcribe.py:241-246,1463-1466``), greedy and random sampling.
  **Parity unpinned** for this part: the reference tests hold no numeric golden vectors at the
  CTranslate2 boundary and the library cannot be run here (SURVEY.md §8c).

Everything computes in float32 (torch CPU for the contractions, NumPy for the search).
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

LOWEST = float(np.finfo(np.float32).min)  # CTranslate2's DisableTokens writes lowest(), not -inf


# --------------------------------------------------------------------------------------------------
# log-mel front end (feature_extractor.py)
# --------------------------------------------------------------------------------------------------
def mel_filters(sr: int = 16000, n_fft: int = 400, n_mels: int = 80) -> np.ndarray:
    """Slaney mel filterbank, float64 math, cast to float32 (feature_extractor.py:24-65, :20-22)."""
    fftfreqs = np.fft.rfftfreq(n=n_fft, d=1.0 / sr)
    mels = np.linspace(0.0, 45.245640471924965, n_mels + 2)
    f_sp = 200.0 / 3
    freqs = f_sp * mels
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    log_t = mels >= min_log_mel
    freqs[log_t] = min_log_hz * np.exp(logstep * (mels[log_t] - min_log_mel))
    fdiff = np.diff(freqs)
    ramps = freqs.reshape(-1, 1) - fftfreqs.reshape(1, -1)
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    weights = np.maximum(0.0, np.minimum(lower, upper))
    weights *= (2.0 / (freqs[2 : n_mels + 2] - freqs[:n_mels]))[:, None]
    return weights.astype(np.float32)


def log_mel(
    waveform: np.ndarray, n_mels: int = 80, padding: int = 160, n_fft: int = 400, hop: int = 160,
    sr: int = 16000, filters: Optional[np.ndarray] = None,
) -> np.ndarray:
    """FeatureExtractor.__call__ restated (feature_extractor.py:198-230): float32 [n_mels, 1+N//hop]."""
    x = np.asarray(waveform, dtype=np.float32)
    if padding:
        x = np.pad(x, (0, padding))
    window = np.hanning(n_fft + 1)[:-1].astype(np.float32)
    xp = np.pad(x, (n_fft // 2, n_fft // 2), mode="reflect")  # stft(center=True), :117-121
    n_frames = 1 + (xp.shape[0] - n_fft) // hop  # :157
    idx = hop * np.arange(n_frames)[:, None] + np.arange(n_fft)[None, :]
    frames = xp[idx] * window  # :170-171
    spec = np.fft.rfft(frames, n=n_fft, axis=-1).astype(np.complex64)  # :189, :221
    mag = np.abs(spec.T[:, :-1]) ** 2  # :222  [201, n_frames-1]
    if filters is None:
        filters = mel_filters(sr, n_fft, n_mels)
    mel = filters @ mag  # :224
    log_spec = np.log10(np.clip(mel, a_min=1e-10, a_max=None))
    log_spec = np.maximum(log_spec, log_spec.max() - 8.0)  # :227 global max over the whole input
    return ((log_spec + 4.0) / 4.0).astype(np.float32)


def pad_or_trim(array: np.ndarray, length: int = 3000) -> np.ndarray:
    """audio.py:111-123 (last axis, zero padding in normalised log-mel space)."""
    if array.shape[-1] > length:
        array = array[..., :length]
    if array.shape[-1] < length:
        pad = [(0, 0)] * array.ndim
        pad[-1] = (0, length - array.shape[-1])
        array = np.pad(array, pad)
    return array


# --------------------------------------------------------------------------------------------------
# network
# --------------------------------------------------------------------------------------------------
@dataclass
class GenerationResult:
    sequences_ids: List[List[int]]
    scores: List[float]
    no_speech_prob: float
    # diagnostics for near-tie analysis in tests (not part of the CT2 surface)
    min_margin: float = float("inf")
    steps: int = 0
    step_margins: Optional[List[float]] = None  # greedy rows: top-1 / top-2 log-prob gap at every step of the best hypothesis


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).float()


class WhisperOracle:
    """float32 Whisper with CTranslate2 decoding semantics."""

    def __init__(self, dims: dict, weights: Dict[str, np.ndarray], tokens: dict,
                 suppress_ids_begin: Optional[Sequence[int]] = None, num_threads: Optional[int] = None, int8_dynamic: bool = False):
        """``int8_dynamic``: bench.py's CPU arm only — every linear layer (and the output embedding) runs as a torch dynamic-int8
        linear (per-tensor int8 weights, activations quantised per call), the closest stand-in available here for the reference's
        ``compute_type="int8"`` CPU path (CTranslate2 itself cannot be installed, SURVEY.md §8c).  Parity tests never set it."""
        if num_threads:
            torch.set_num_threads(num_threads)
        self.dims = dict(dims)
        self.tok = dict(tokens)
        self.w = {k: _t(v) for k, v in weights.items()}
        self.q: Dict[str, torch.nn.Module] = {}
        if int8_dynamic:
            self._quantize_linears()
        self.n_head = self.dims["n_text_head"]
        self.n_audio_head = self.dims["n_audio_head"]
        self.n_vocab = self.dims["n_vocab"]
        # CT2 reads these two lists from the converted model's config.json ("suppress_ids_begin" = [" ", eot]).
        self.suppress_ids_begin = list(suppress_ids_begin) if suppress_ids_begin is not None else [220, self.tok["eot"]]

    # ---- encoder ---------------------------------------------------------------------------------
    def _ln(self, x, prefix):
        return F.layer_norm(x, (x.shape[-1],), self.w[prefix + ".weight"], self.w[prefix + ".bias"], 1e-5)

    def _lin(self, x, prefix, bias=True):
        if prefix in self.q:
            return self.q[prefix](x)
        return F.linear(x, self.w[prefix + ".weight"], self.w.get(prefix + ".bias") if bias else None)

    def _quantize_linears(self):
        import torch.ao.nn.quantized.dynamic as nnqd

        def make(wt, bias):
            lin = torch.nn.Linear(wt.shape[1], wt.shape[0], bias=bias is not None)
            lin.weight = torch.nn.Parameter(wt, requires_grad=False)
            if bias is not None:
                lin.bias = torch.nn.Parameter(bias, requires_grad=False)
            lin.qconfig = torch.ao.quantization.default_dynamic_qconfig
            return nnqd.Linear.from_float(lin)

        for name in list(self.w):
            if name.endswith(".weight") and self.w[name].ndim == 2 and (".attn." in name or ".cross_attn." in name or ".mlp." in name):
                prefix = name[: -len(".weight")]
                self.q[prefix] = make(self.w[name], self.w.get(prefix + ".bias"))
        self.q["__logits__"] = make(self.w["decoder.token_embedding.weight"], None)

    @staticmethod
    def _split_heads(x, n_head):
        b, t, d = x.shape
        return x.view(b, t, n_head, d // n_head).permute(0, 2, 1, 3)

    def _mha(self, q, k, v, n_head, mask=None):
        q, k, v = (self._split_heads(z, n_head) for z in (q, k, v))
        scale = (q.shape[-1]) ** -0.5
        att = (q @ k.transpose(-1, -2)) * scale
        if mask is not None:
            att = att + mask
        att = torch.softmax(att, dim=-1)
        out = att @ v
        b, h, t, hd = out.shape
        return out.permute(0, 2, 1, 3).reshape(b, t, h * hd), att

    @torch.no_grad()
    def encode(self, features: np.ndarray) -> torch.Tensor:
        """[B, n_mels, 3000] float32 -> [B, 1500, d] (CT2 Whisper.encode, transcribe.py:209,1400)."""
        x = _t(features)
        if x.ndim == 2:
            x = x[None]
        x = F.gelu(F.conv1d(x, self.w["encoder.conv1.weight"], self.w["encoder.conv1.bias"], padding=1))
        x = F.gelu(F.conv1d(x, self.w["encoder.conv2.weight"], self.w["encoder.conv2.bias"], stride=2, padding=1))
        x = x.permute(0, 2, 1) + self.w["encoder.positional_embedding"][: x.shape[-1]]
        for i in range(self.dims["n_audio_layer"]):
            p = f"encoder.blocks.{i}"
            h = self._ln(x, p + ".attn_ln")
            a, _ = self._mha(self._lin(h, p + ".attn.query"), self._lin(h, p + ".attn.key", bias=False),
                             self._lin(h, p + ".attn.value"), self.n_audio_head)
            x = x + self._lin(a, p + ".attn.out")
            h = self._ln(x, p + ".mlp_ln")
            x = x + self._lin(F.gelu(self._lin(h, p + ".mlp.0")), p + ".mlp.2")
        return self._ln(x, "encoder.ln_post")

    # ---- decoder ---------------------------------------------------------------------------------
    @torch.no_grad()
    def cross_kv(self, enc: torch.Tensor):
        out = []
        for i in range(self.dims["n_text_layer"]):
            p = f"decoder.blocks.{i}.cross_attn"
            out.append((self._lin(enc, p + ".key", bias=False), self._lin(enc, p + ".value")))
        return out

    @torch.no_grad()
    def decoder_forward(self, tokens: torch.Tensor, offset: int, cache: list, xkv: list, row2chunk: torch.Tensor,
                        want_cross_att: bool = False):
        """tokens [R, n] at positions offset..offset+n-1; cache[l] = (K,V) [R, offset, d] or None.
        Returns logits [R, n, V] and updates cache in place."""
        w = self.w
        n = tokens.shape[1]
        x = w["decoder.token_embedding.weight"][tokens] + w["decoder.positional_embedding"][offset : offset + n]
        mask = None
        if n > 1:
            mask = torch.full((n, offset + n), 0.0)
            mask[:, offset:] = torch.triu(torch.full((n, n), float("-inf")), diagonal=1)
        cross_atts = []
        for i in range(self.dims["n_text_layer"]):
            p = f"decoder.blocks.{i}"
            h = self._ln(x, p + ".attn_ln")
            k_new = self._lin(h, p + ".attn.key", bias=False)
            v_new = self._lin(h, p + ".attn.value")
            if cache[i] is None:
                k_all, v_all = k_new, v_new
            else:
                k_all = torch.cat([cache[i][0], k_new], dim=1)
                v_all = torch.cat([cache[i][1], v_new], dim=1)
            cache[i] = (k_all, v_all)
            a, _ = self._mha(self._lin(h, p + ".attn.query"), k_all, v_all, self.n_head, mask)
            x = x + self._lin(a, p + ".attn.out")
            h = self._ln(x, p + ".cross_attn_ln")
            xk, xv = xkv[i]
            if xk.shape[0] == 1:  # every row reads the same chunk: broadcast instead of materialising one K/V copy per beam
                xk_r, xv_r = xk.expand(x.shape[0], -1, -1), xv.expand(x.shape[0], -1, -1)
            else:
                xk_r, xv_r = xk[row2chunk], xv[row2chunk]
            a, att = self._mha(self._lin(h, p + ".cross_attn.query"), xk_r, xv_r, self.n_head)
            if want_cross_att:
                cross_atts.append(att)
            x = x + self._lin(a, p + ".cross_attn.out")
            h = self._ln(x, p + ".mlp_ln")
            x = x + self._lin(F.gelu(self._lin(h, p + ".mlp.0")), p + ".mlp.2")
        x = self._ln(x, "decoder.ln")
        # "decoder.output_projection.weight" (tests of quantised engines only): an output embedding that differs from the input one
        out_w = w.get("decoder.output_projection.weight", w["decoder.token_embedding.weight"])
        logits = self.q["__logits__"](x) if "__logits__" in self.q else x @ out_w.t()
        return (logits, cross_atts) if want_cross_att else logits

    # ---- logits processors (CT2 semantics, CPU ordering: DisableTokens writes immediately) --------
    def _process_logits(self, logits: np.ndarray, step: int, histories: List[List[int]], o: dict) -> None:
        """In place on [R, V] float32.  `step` counts generated tokens (sample_begin == 0)."""
        tok = self.tok
        V = logits.shape[1]
        rp = o["repetition_penalty"]
        if rp != 1.0:
            for r, h in enumerate(histories):
                if h:
                    ids = np.unique(np.asarray(h, dtype=np.int64))
                    vals = logits[r, ids]
                    logits[r, ids] = np.where(vals < 0, vals * np.float32(rp), vals / np.float32(rp))
        ng = o["no_repeat_ngram_size"]
        if ng > 0:
            for r, h in enumerate(histories):
                if len(h) >= ng:
                    prefix = h[len(h) - ng + 1 :] if ng > 1 else []
                    for s in range(len(h) - ng + 1):
                        if h[s : s + ng - 1] == prefix:
                            logits[r, h[s + ng - 1]] = LOWEST
        if o["suppress_ids"].size:
            logits[:, o["suppress_ids"]] = LOWEST
        if o["suppress_blank"] and step == 0:
            logits[:, self.suppress_ids_begin] = LOWEST
        if o["timestamp_rules"]:
            ts0, eot = tok["timestamp_begin"], tok["eot"]
            for r, h in enumerate(histories):
                row = logits[r]
                row[tok["no_timestamps"]] = LOWEST
                if step == 0:
                    row[:ts0] = LOWEST  # first sampled token must be a timestamp
                    mi = o["max_initial_timestamp_index"]
                    if mi is not None and mi >= 0:
                        row[ts0 + mi + 1 :] = LOWEST
                    continue
                last_ts = h[-1] >= ts0
                penult_ts = len(h) < 2 or h[-2] >= ts0
                if last_ts:
                    if penult_ts:
                        row[ts0:] = LOWEST  # after a closed pair: text (or EOT) only
                    else:
                        row[:eot] = LOWEST  # a lone timestamp must be followed by a timestamp or EOT
                stamps = [t for t in h if t >= ts0]
                if stamps:
                    # timestamps may not decrease; force non-zero segment length unless closing a segment
                    t_last = stamps[-1] if (last_ts and not penult_ts) else stamps[-1] + 1
                    row[ts0:t_last] = LOWEST
                # if total timestamp mass beats every single text token, force a timestamp
                m = row.max()
                lse = m + np.log(np.exp((row - m).astype(np.float64)).sum())
                lp = row.astype(np.float64) - lse
                ts_lp = lp[ts0:]
                mt = ts_lp.max()
                ts_logprob = mt + np.log(np.exp(ts_lp - mt).sum()) if np.isfinite(mt) and mt > LOWEST / 2 else -np.inf
                if ts_logprob > lp[:ts0].max():
                    row[:ts0] = LOWEST

    @staticmethod
    def _log_softmax(logits: np.ndarray) -> np.ndarray:
        x = logits.astype(np.float64)
        m = x.max(axis=-1, keepdims=True)
        lse = m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True))
        return (x - lse).astype(np.float32)

    # ---- generate --------------------------------------------------------------------------------
    @torch.no_grad()
    def generate(self, enc: torch.Tensor, prompts: Sequence[Sequence[int]], *, beam_size: int = 5, patience: float = 1.0,
                 num_hypotheses: int = 1, length_penalty: float = 1.0, repetition_penalty: float = 1.0,
                 no_repeat_ngram_size: int = 0, max_length: int = 448, return_scores: bool = True,
                 return_no_speech_prob: bool = True, max_initial_timestamp_index: int = 50, suppress_blank: bool = True,
                 suppress_tokens: Optional[Sequence[int]] = (-1,), sampling_topk: int = 1, sampling_temperature: float = 1.0,
                 seed: int = 0, fake_logits=None, trace: Optional[list] = None) -> List[GenerationResult]:
        tok = self.tok
        B = enc.shape[0] if enc is not None else len(prompts)
        if len(prompts) != B:
            raise ValueError("one prompt per batch item is required")
        P = len(prompts[0])
        sot_index = None
        for p in prompts:
            if len(p) != P:
                raise ValueError("all prompts in a batch must have the same length")
            if tok["sot"] not in p:
                raise ValueError("<|startoftranscript|> token was not found in the prompt")
            s = list(p).index(tok["sot"])
            if sot_index is None:
                sot_index = s
            elif s != sot_index:
                raise ValueError("<|startoftranscript|> must be at the same position in all prompts")
        if P >= max_length:
            return [GenerationResult([[]], [0.0], 0.0) for _ in range(B)]
        sup = [t for t in (suppress_tokens or []) if t >= 0]
        if suppress_tokens is not None and -1 in suppress_tokens:
            sup += list(self.dims.get("suppress_ids", []))
        o = dict(
            repetition_penalty=float(repetition_penalty), no_repeat_ngram_size=int(no_repeat_ngram_size),
            suppress_ids=np.asarray(sorted(set(sup)), dtype=np.int64), suppress_blank=bool(suppress_blank),
            timestamp_rules=tok["no_timestamps"] not in prompts[0],
            max_initial_timestamp_index=int(max_initial_timestamp_index),
        )
        n_layer = self.dims["n_text_layer"]
        xkv = self.cross_kv(enc) if fake_logits is None else None
        prompt_t = torch.tensor([list(p) for p in prompts], dtype=torch.long)
        row2chunk = torch.arange(B)
        cache: list = [None] * n_layer
        no_speech = [0.0] * B
        if fake_logits is None and P > 1:
            lg = self.decoder_forward(prompt_t[:, : P - 1], 0, cache, xkv, row2chunk)
            if return_no_speech_prob and sot_index < P - 1:
                pr = torch.softmax(lg[:, sot_index].double(), dim=-1)
                no_speech = [float(pr[b, tok["no_speech"]]) for b in range(B)]
        need_ns_first = return_no_speech_prob and sot_index == P - 1
        max_steps = max_length - P

        def forward(tokens_rows: List[int], step: int, r2c: torch.Tensor, hist):
            if fake_logits is not None:
                return fake_logits(tokens_rows, step, hist)
            t = torch.tensor(tokens_rows, dtype=torch.long)[:, None]
            return self.decoder_forward(t, P - 1 + step, cache, xkv, r2c)[:, 0].numpy().copy()

        def reorder(idx: List[int]):
            if fake_logits is not None:
                return
            ii = torch.tensor(idx, dtype=torch.long)
            for i in range(n_layer):
                cache[i] = (cache[i][0][ii], cache[i][1][ii])

        results: List[GenerationResult] = []
        if beam_size <= 1:
            results = self._greedy(B, prompts, forward, reorder, o, max_steps, num_hypotheses, length_penalty,
                                   sampling_topk, sampling_temperature, seed, need_ns_first, no_speech, trace,
                                   has_cache=(fake_logits is None and P > 1))
        else:
            results = self._beam(B, prompts, forward, reorder, o, max_steps, beam_size, patience, num_hypotheses,
                                 length_penalty, need_ns_first, no_speech, trace)
        if not return_no_speech_prob:
            for r in results:
                r.no_speech_prob = 0.0
        return results

    def _finalize_score(self, cum: float, length: int, lp: float) -> float:
        if lp == 0:
            return float(cum)
        denom = float(length) ** lp
        with np.errstate(divide="ignore", invalid="ignore"):
            return float(np.float32(cum) / np.float32(denom)) if denom != 0 else float(np.float32(cum) / np.float32(0.0))

    # greedy / random sampling (CT2 GreedySearch; beam_size == 1)
    def _greedy(self, B, prompts, forward, reorder, o, max_steps, num_hyp, lp, topk, temperature, seed, need_ns_first,
                no_speech, trace, has_cache=False):
        tok = self.tok
        eot = tok["eot"]
        H = max(1, num_hyp)
        R = B * H
        rows_chunk = [b for b in range(B) for _ in range(H)]
        r2c = torch.tensor(rows_chunk, dtype=torch.long)
        if H > 1 and has_cache:
            reorder(rows_chunk)  # one copy of the prompt state per hypothesis
        last = [prompts[b][-1] for b in rows_chunk]
        hist: List[List[int]] = [[] for _ in range(R)]
        cum = [0.0] * R
        done = [False] * R
        margin = [float("inf")] * R
        step_margin: List[List[float]] = [[] for _ in range(R)]
        steps = 0
        for step in range(max_steps):
            logits = forward(last, step, r2c, hist)
            if step == 0 and need_ns_first:
                pr = self._softmax64(logits)
                for r in range(R):
                    no_speech[rows_chunk[r]] = float(pr[r, tok["no_speech"]])
            self._process_logits(logits, step, hist, o)
            logp = self._log_softmax(logits)
            if trace is not None:
                trace.append(dict(step=step, logits=logits.copy(), logp=logp.copy()))
            steps += 1
            for r in range(R):
                if done[r]:
                    continue
                if topk == 1:
                    order = np.argsort(-logp[r], kind="stable")[:2]
                    t = int(order[0])
                    margin[r] = min(margin[r], float(logp[r, order[0]] - logp[r, order[1]]))
                    step_margin[r].append(float(logp[r, order[0]] - logp[r, order[1]]))
                    sc = float(logp[r, t])
                else:
                    t, sc = self._sample(logp[r], topk, temperature, seed, r, step)
                cum[r] += sc
                if t == eot or step + 1 == max_steps:
                    done[r] = True
                    if t != eot:
                        hist[r].append(t)
                else:
                    hist[r].append(t)
                last[r] = t
            if all(done):
                break
        out = []
        for b in range(B):
            rows = [r for r in range(R) if rows_chunk[r] == b]
            cands = [(self._finalize_score(cum[r], len(hist[r]), lp), r) for r in rows]
            cands.sort(key=lambda x: (-x[0] if not math.isnan(x[0]) else float("inf"), x[1]))
            out.append(GenerationResult([hist[r] for _, r in cands], [s for s, _ in cands], no_speech[b],
                                        min(margin[r] for r in rows), steps, step_margin[cands[0][1]] if topk == 1 else None))
        return out

    @staticmethod
    def _softmax64(logits: np.ndarray) -> np.ndarray:
        x = logits.astype(np.float64)
        x = x - x.max(axis=-1, keepdims=True)
        e = np.exp(x)
        return e / e.sum(axis=-1, keepdims=True)

    @staticmethod
    def gumbel_noise(seed: int, row: int, step: int, n: int) -> np.ndarray:
        """Counter-based noise shared with the CUDA sampler (csrc/search.cu: gumbel_u32)."""
        # 23 random bits + 0.5 is exact in float32 and keeps u strictly inside (0, 1)
        u = (WhisperOracle.gumbel_bits(seed, row, step, n).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 8388608.0)
        return (-np.log(-np.log(u))).astype(np.float32)

    @staticmethod
    def gumbel_bits(seed: int, row: int, step: int, n: int) -> np.ndarray:
        """The 23-bit integers u * 2^23 - 0.5 behind gumbel_noise, for token ids 0..n-1."""
        M = (1 << 64) - 1
        base = (seed * 0xBF58476D1CE4E5B9 + row * 0x94D049BB133111EB + step * 0xD6E8FEB86659FD93) & M
        with np.errstate(over="ignore"):
            x = np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(base)  # wraps mod 2^64
            x ^= x >> np.uint64(30)
            x = x * np.uint64(0xBF58476D1CE4E5B9)
            x ^= x >> np.uint64(27)
            x = x * np.uint64(0x94D049BB133111EB)
            x ^= x >> np.uint64(31)
        return x >> np.uint64(41)

    def _sample(self, logp_row: np.ndarray, topk: int, temperature: float, seed: int, row: int, step: int):
        """Random sampling as Gumbel-max over logp/T (distributionally equal to CT2's multinomial;
        the returned score is the tempered log-prob of the draw, as CT2's RandomSampler gathers it)."""
        with np.errstate(over="ignore"):
            z = logp_row / np.float32(temperature) if temperature != 1 else logp_row.copy()
        if topk > 0:
            kth = np.partition(z, -topk)[-topk]
            z = np.where(z >= kth, z, np.float32(LOWEST))
        g = z + self.gumbel_noise(seed, row, step, z.shape[0])
        g = np.where(z <= LOWEST / 2, np.float32(LOWEST), g)
        t = int(np.argmax(g))
        return t, float(z[t])

    # beam search (CT2 BeamSearch: 2K candidates, patience, finished hypotheses replaced by secondary candidates)
    def _beam(self, B, prompts, forward, reorder, o, max_steps, K, patience, num_hyp, lp, need_ns_first, no_speech, trace):
        tok = self.tok
        eot = tok["eot"]
        V = self.n_vocab
        ncand = 2 * K
        max_cand = int(math.floor(K * patience + 0.5))  # std::round: halves away from zero
        allow_early_exit = patience == 1 and lp == 0
        # per chunk state
        hist = [[[]] for _ in range(B)]  # hist[b][k] -> tokens ; starts unexpanded with one row per chunk
        cum = [[0.0] for _ in range(B)]
        last = [[prompts[b][-1]] for b in range(B)]
        finished: List[List[Tuple[float, List[int]]]] = [[] for _ in range(B)]
        done = [False] * B
        margin = [float("inf")] * B
        rows_src = list(range(B))  # cache row index for each (b,k) flattened, in current cache
        steps = 0
        for step in range(max_steps):
            live = [b for b in range(B)]
            nb = [len(hist[b]) for b in range(B)]
            rows = [(b, k) for b in range(B) for k in range(nb[b])]
            r2c = torch.tensor([b for b, _ in rows], dtype=torch.long)
            logits = forward([last[b][k] for b, k in rows], step, r2c, [hist[b][k] for b, k in rows])
            if step == 0 and need_ns_first:
                pr = self._softmax64(logits)
                for r, (b, _) in enumerate(rows):
                    no_speech[b] = float(pr[r, tok["no_speech"]])
            self._process_logits(logits, step, [hist[b][k] for b, k in rows], o)
            logp = self._log_softmax(logits)
            if trace is not None:
                trace.append(dict(step=step, logits=logits.copy(), logp=logp.copy(), rows=list(rows)))
            steps += 1
            is_last = step + 1 == max_steps
            new_index: List[int] = []
            r0 = 0
            for b in range(B):
                n = nb[b]
                block = logp[r0 : r0 + n] + np.asarray(cum[b], dtype=np.float32)[:, None]
                flat = block.reshape(-1)
                # top 2K, ties -> lower flat index
                part = np.argpartition(-flat, min(ncand, flat.size - 1))[: ncand + 1]
                order = part[np.lexsort((part, -flat[part]))][: ncand + 1]
                if order.size > ncand:
                    margin[b] = min(margin[b], float(flat[order[ncand - 1]] - flat[order[ncand]])) if not done[b] else margin[b]
                    gaps = np.diff(-flat[order[:ncand]])
                    if gaps.size and not done[b]:
                        margin[b] = min(margin[b], float(gaps.min()))
                order = order[:ncand]
                cand_beam = (order // V).tolist()
                cand_tok = (order % V).tolist()
                cand_score = flat[order].tolist()
                new_hist, new_cum, new_last, src = [], [], [], []
                secondary = K
                top_finished = False
                for k in range(K):
                    nxt = k
                    t = cand_tok[k]
                    if (t == eot or is_last) and not done[b]:
                        if k == 0:
                            top_finished = True
                        seq = hist[b][cand_beam[k]] + ([] if t == eot else [t])
                        finished[b].append((cand_score[k], seq))
                        for j in range(secondary, ncand):
                            if cand_tok[j] != eot:
                                nxt = j
                                secondary = j + 1
                                break
                    new_hist.append(hist[b][cand_beam[nxt]] + [cand_tok[nxt]])
                    new_cum.append(cand_score[nxt])
                    new_last.append(cand_tok[nxt])
                    src.append(r0 + cand_beam[nxt])
                if not done[b]:
                    if is_last:
                        done[b] = True
                    elif allow_early_exit:
                        done[b] = top_finished and len(finished[b]) >= num_hyp
                    else:
                        done[b] = len(finished[b]) >= max_cand
                hist[b], cum[b], last[b] = new_hist, new_cum, new_last
                new_index += src
                r0 += n
            if all(done):
                break
            reorder(new_index)
        out = []
        for b in range(B):
            fin = [(self._finalize_score(s, len(seq), lp), i, seq) for i, (s, seq) in enumerate(finished[b])]
            fin.sort(key=lambda x: (-x[0] if not math.isnan(x[0]) else float("inf"), x[1]))
            fin = fin[: max(1, num_hyp)]
            out.append(GenerationResult([s for _, _, s in fin], [sc for sc, _, _ in fin], no_speech[b], margin[b], steps))
        return out

    # ---- language detection (CT2 Whisper.detect_language, transcribe.py:215,1193,1823) -------------
    @torch.no_grad()
    def detect_language(self, enc: torch.Tensor) -> List[List[Tuple[int, float]]]:
        tok = self.tok
        B = enc.shape[0]
        xkv = self.cross_kv(enc)
        cache: list = [None] * self.dims["n_text_layer"]
        t = torch.full((B, 1), tok["sot"], dtype=torch.long)
        lg = self.decoder_forward(t, 0, cache, xkv, torch.arange(B))[:, 0]
        ids = list(range(tok["lang_begin"], tok["lang_begin"] + tok["num_languages"]))
        pr = torch.softmax(lg[:, ids].double(), dim=-1).numpy()
        out = []
        for b in range(B):
            order = np.argsort(-pr[b], kind="stable")
            out.append([(ids[i], float(pr[b, i])) for i in order])
        return out

    # ---- word-level alignment (CT2 Whisper.align; consumer at transcribe.py:1698-1766) ---------------------------------
    def default_alignment_heads(self) -> List[Tuple[int, int]]:
        """Every head of the last half of the decoder layers (OpenAI Whisper's default when a checkpoint lists none)."""
        L, H = self.dims["n_text_layer"], self.dims["n_text_head"]
        return [(l, h) for l in range(L // 2, L) for h in range(H)]

    @torch.no_grad()
    def align(self, enc: torch.Tensor, start_sequence: Sequence[int], text_tokens: Sequence[Sequence[int]], num_frames,
              median_filter_width: int = 7, alignment_heads: Optional[Sequence[Tuple[int, int]]] = None) -> List["AlignmentResult"]:
        """Restated (parity unpinned, DESIGN.md §7): teacher-force ``start_sequence + [no_timestamps] + text + [eot]``, take
        the cross-attention probabilities of the alignment heads over the first ``num_frames // 2`` encoder positions,
        normalise over the token axis (population std), median-filter along time (reflect padding), average the heads, keep
        the rows of the inputs that predict ``text + [eot]`` (drop the start-sequence rows and the eot input row: the consumer
        indexes word boundaries up to len(text), transcribe.py:1744-1746), DTW on the negated matrix.  ``text_token_probs[t]`` is the full-vocabulary
        softmax probability of text token t at the position that predicts it."""
        tok = self.tok
        heads = list(alignment_heads) if alignment_heads is not None else self.default_alignment_heads()
        out = []
        for b, toks in enumerate(text_tokens):
            nf = int(num_frames[b] if isinstance(num_frames, (list, tuple)) else num_frames)
            start = list(start_sequence) + [tok["no_timestamps"]]
            seq = start + list(toks) + [tok["eot"]]
            xkv = self.cross_kv(enc[b : b + 1])
            cache: list = [None] * self.dims["n_text_layer"]
            logits, atts = self.decoder_forward(torch.tensor([seq], dtype=torch.long), 0, cache, xkv, torch.zeros(1, dtype=torch.long),
                                                want_cross_att=True)
            probs = torch.softmax(logits[0].double(), dim=-1)
            tprobs = [float(probs[len(start) - 1 + t, toks[t]]) for t in range(len(toks))]
            w = torch.stack([atts[l][0, h] for l, h in heads]).double()[:, :, : max(1, nf // 2)]
            mean = w.mean(dim=-2, keepdim=True)
            std = w.std(dim=-2, keepdim=True, unbiased=False)
            w = (w - mean) / std
            w = median_filter(w.numpy(), median_filter_width)
            m = w.mean(axis=0)[len(start_sequence) : -1]  # inputs <|notimestamps|>, text[0..n-2], text[n-1]: the rows predicting text + eot
            ti, fi = dtw(-m)
            out.append(AlignmentResult(alignments=list(zip(ti.tolist(), fi.tolist())), text_token_probs=tprobs))
        return out


@dataclass
class AlignmentResult:
    alignments: List[Tuple[int, int]]
    text_token_probs: List[float]


def median_filter(x: np.ndarray, width: int) -> np.ndarray:
    """Median over a sliding window of odd `width` along the last axis, reflect padding; rows shorter than the padding are
    returned unchanged."""
    pad = width // 2
    if pad == 0 or x.shape[-1] <= pad:
        return x
    xp = np.pad(x, [(0, 0)] * (x.ndim - 1) + [(pad, pad)], mode="reflect")
    win = np.lib.stride_tricks.sliding_window_view(xp, width, axis=-1)
    return np.sort(win, axis=-1)[..., pad]


def dtw(cost_in: np.ndarray):
    """Monotone path of minimal accumulated cost through [N, M] (moves: diagonal, down, right; ties prefer the right move
    unless the diagonal is strictly best, then the down move)."""
    N, M = cost_in.shape
    cost = np.full((N + 1, M + 1), np.inf)
    trace = np.full((N + 1, M + 1), -1, dtype=np.int64)
    cost[0, 0] = 0.0
    for j in range(1, M + 1):
        for i in range(1, N + 1):
            c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
            if c0 < c1 and c0 < c2:
                c, t = c0, 0
            elif c1 < c0 and c1 < c2:
                c, t = c1, 1
            else:
                c, t = c2, 2
            cost[i, j] = cost_in[i - 1, j - 1] + c
            trace[i, j] = t
    i, j = N, M
    trace[0, :] = 2
    trace[:, 0] = 1
    ti, fi = [], []
    while i > 0 or j > 0:
        ti.append(i - 1)
        fi.append(j - 1)
        t = trace[i, j]
        if t == 0:
            i -= 1
            j -= 1
        elif t == 1:
            i -= 1
        else:
            j -= 1
    return np.array(ti[::-1]), np.array(fi[::-1])
