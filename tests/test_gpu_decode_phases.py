"""Every grid phase of the many-row decode step (bstep_kernel) and both standalone decoder attention kernels (dec_self_attn_kernel,
ds_cross_attn_kernel) against float64, on the inputs the kernels actually received.

The logits tests (test_gpu_step_logits.py) bound a whole step at 0.05, which cannot see one dropped or doubled key among 1500
flat cross-attention scores (about |v| / 1500 before the output projection).  Here:

* phases: debug_step_logits with B2W_STEP=bstep and B2W_BSTEP_STOP=p stops every step of a forced decode after grid phase p,
  which leaves everything phase p reads (the caches of earlier steps included) as a full run leaves it; debug_fetch then reads
  the workspace and the phase is restated in float64 on those fp16 / fp32 operands.  A residual GEMM updates x in place, so its
  input comes from the run stopped at p - 1 (the kernel is bit-reproducible).  `pytest -k phase -s` prints one line per phase,
  which bisects a wrong kernel.
* probes: with the query weights zeroed every score is 0, so attention is the plain mean of V over exactly the visible keys;
  with one-hot queries (a target key whose score beats every other by >= 16) the output is v_target to fp16 rounding.
* sensitivity: for every attention check on random or model-produced inputs, removing one key (key 0, the row's own position,
  key 1499, the first key of each cross-attention split and of each 16-key self-attention block) from the float64 reference
  moves it by more than the bound, so each bound is shown to see a dropped key.
* a residual row offset (|mean| / std of about 8 and 32) checks the deferred LayerNorm against its error model: the kernel
  stages the raw residual in fp16, so y = LN(x) W + b is off by up to c 2^-11 rstd sqrt(sum_k W_nk^2 x_k^2) plus fp32 terms.

Bounds, elementwise; h(y) is half the fp16 spacing at |y| (the rounding of an fp16 output), V the largest |v| of the case.
Largest measured error and error / bound ratio on an NVIDIA H100 80GB HBM3 (700 W power limit):

    embed                        bit-exact
    split-K raw sums             ERR_SUM sum_k |W_nk x_k| + 1e-6                      5.4e-6  (ratio 0.27)
    row statistics               ERR_SUM sum |x| (sum x^2) + 1e-6                     7.3e-4  (0.43)
    k, v cache entries, h16      h(y) + ERR_LN_REL max|y|                             1.9e-3  (0.82)
    residual GEMMs               ERR_SUM (sum_k |W_nk a_k| + |x|) + 1e-6              1.9e-6  (0.15)
    bstep attention              h(o) + u sum_j p_j |v_j - o| + ERR_ATTN_REL V        9.8e-4  (0.97)
        (u = 2^-11: the phases round the probabilities to fp16 before P V)
    zero-query probes            h(o) + ERR_UNIFORM_REL V                             9.6e-4  (0.95)
    one-hot probes               h(v_target) + 1e-4                                   0       (0)
    standalone kernels, random   h(o) + ERR_HOOK_REL V                                4.9e-4  (0.83)
    final LN                     h(y) + 1e-5 |y| + 1e-6                               9.8e-4  (0.98)
    logits                       ERR_SUM sum_k |E_vk xn_k| + 1e-4                     5.2e-5  (0.35)
    row offset (8 and 32 sigma)  4 u rstd sqrt(sum_k W_nk^2 x_k^2)
                                 + (2^-10 + 4 u |mean| rstd / sqrt(d)) |y| + 1e-5     3.3e-2  (0.54)

The attention and final-LN ratios near 1 are the fp16 rounding of the output itself, which no bound can go below.
"""
import os

import numpy as np
import pytest
import torch
from scipy.special import erf

from faster_whisper_b200 import engine
from faster_whisper_b200.config import special_tokens
from faster_whisper_b200.synthetic import custom_dims, make_weights
from test_gpu_step_logits import features_for, forced_inputs, make_engine, prefix_prompt

ERR_SUM = 5e-7
ERR_LN_REL = 1e-4
ERR_ATTN_REL = 2e-5   # bstep's attention phases, on top of their fp16-probability term
ERR_HOOK_REL = 2e-5   # the standalone kernels on random inputs
ERR_UNIFORM_REL = 1e-5
T_AUDIO = 1500
SPLITS = 7
F16_U = 2.0 ** -11


# ---- pure NumPy helpers (tested on the CPU below) -------------------------------------------------------------------
def key_slots(P, parents, t, b, k, K):
    """Slot of every key 0 .. pos (pos = P - 1 + t) that row (chunk b, slot k) reads at step t of a forced decode: the prompt's keys
    sit in slot 0, the key of step s < t in the slot the row's ancestor held at step s, its own key in slot k."""
    pos = P - 1 + t
    out = np.zeros(pos + 1, np.int64)
    a = k
    for s in range(t, -1, -1):
        out[P - 1 + s] = a
        if s > 0 and parents is not None:
            a = int(parents[s, b, a])
    return out


def xkv_swizzle(x):
    """[..., T, 64] <-> the encoder output's stored layout, whose 16-byte chunk c of key t holds chunk c ^ (t & 7) (an involution)."""
    T = x.shape[-2]
    t = np.arange(T)
    y = x.reshape(x.shape[:-1] + (8, 8))
    return y[..., t[:, None], np.arange(8)[None, :] ^ (t[:, None] & 7), :].reshape(x.shape)


def bs_group(NB, KA, G, nb):
    base, extra = G // NB, G % NB
    g0 = nb * base + min(nb, extra)
    return g0, min(base + 1 if nb < extra else base, KA)


def split_k_sum(parts, n_cols, KA):
    """GEMM output [R, n_cols] from the CTAs' partial tiles parts [G, R, 128]: n-block nb summed over its CTAs g0 .. g0 + gn - 1
    in CTA order, in fp32 (bs_group and bs_ordered_sum in csrc/bstep.cu)."""
    G, R, _ = parts.shape
    NB = (n_cols + 127) // 128
    out = np.zeros((R, NB * 128), np.float32)
    for nb in range(NB):
        g0, gn = bs_group(NB, KA, G, nb)
        acc = parts[g0].astype(np.float32).copy()
        for i in range(1, gn):
            acc = (acc + parts[g0 + i]).astype(np.float32)
        out[:, nb * 128:(nb + 1) * 128] = acc
    return out[:, :n_cols]


def ordered_rows_sum(stpart):
    """sum(x), sum(x^2) per row from the per-k-atom partials [KA, R, 2], added in k order in fp32."""
    acc = stpart[0].astype(np.float32).copy()
    for k in range(1, stpart.shape[0]):
        acc = (acc + stpart[k]).astype(np.float32)
    return acc


def attention(q, K, V, drop=None):
    """float64 softmax(q K^T) V, q [..., 64] already scaled; K, V [..., T, 64]; `drop` removes key index drop."""
    q, K, V = (np.asarray(a, np.float64) for a in (q, K, V))
    if drop is not None:
        K, V = np.delete(K, drop, axis=-2), np.delete(V, drop, axis=-2)
    s = np.einsum("...e,...te->...t", q, K)
    s -= s.max(-1, keepdims=True)
    p = np.exp(s)
    return np.einsum("...t,...te->...e", p / p.sum(-1, keepdims=True), V)


def p_rounding_term(q, K, V):
    """u sum_j p_j |v_j - o|: the most that rounding every probability to fp16 (unit roundoff u = 2^-11, as bstep's attention
    phases do before P V) can move the output, to first order."""
    q, K, V = (np.asarray(a, np.float64) for a in (q, K, V))
    s = np.einsum("...e,...te->...t", q, K)
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    o = np.einsum("...t,...te->...e", p, V)
    return F16_U * np.einsum("...t,...te->...e", p, np.abs(V - o[..., None, :]))


def gelu(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def fp16_ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float16)).astype(np.float64)


def report(label, err, bound):
    e, b = float(np.max(err)) if np.size(err) else 0.0, float(np.max(bound)) if np.size(bound) else 0.0
    ratio = float(np.max(err / bound)) if np.size(err) else 0.0
    print("[decode phases] %-46s max err %.3e  bound %.3e  ratio %.3f" % (label, e, b, ratio), flush=True)
    assert np.all(np.isfinite(err)), (label, "non-finite")
    assert ratio <= 1.0, (label, e, b)


def half_ulp(x):
    """Half the fp16 spacing at |x|: the rounding of an fp16 output."""
    return 0.5 * fp16_ulp(x)


def check_sensitive(label, ref_fn, keys, bound):
    """Removing any one of `keys` from the reference moves it by more than the (elementwise) bound for some element."""
    base = ref_fn(None)
    for j in keys:
        moved = np.abs(ref_fn(j) - base)
        assert (moved > bound).any(), (label, "dropping key", j, "moves no element by more than its bound; largest move",
                                       float(moved.max()))


def split_starts():
    return [T_AUDIO * s // SPLITS for s in range(SPLITS)]


# ---- effective weights: what the kernels multiply with ---------------------------------------------------------------
def _quant(w16):
    """q * scale of fp16 rows, per output channel (ds_quant_rows_kernel), in float64."""
    w = w16.astype(np.float32)
    mx = np.abs(w).max(axis=1, keepdims=True)
    sc = np.where(mx > 0, mx / np.float32(127.0), np.float32(1.0)).astype(np.float32)
    return np.clip(np.rint(w / sc), -127, 127).astype(np.float64) * sc.astype(np.float64)


def effective(w, names, biases, ln=None, int8=False):
    """(W [N, K] float64 as the kernel multiplies, fp32 bias as float64) of the stacked matrices `names`, with the LayerNorm `ln`
    folded in as the engine folds it (fold_ln: W * gamma in fp32, then fp16; bias + W beta)."""
    W = np.concatenate([w[n].astype(np.float32) for n in names])
    b = np.concatenate([w[n].astype(np.float64) if n in w else np.zeros(w[m].shape[0]) for n, m in zip(biases, names)])
    if ln is not None:
        g, beta = w[ln + ".weight"].astype(np.float32), w[ln + ".bias"].astype(np.float64)
        b = (b + W.astype(np.float64) @ beta).astype(np.float32).astype(np.float64)
        W = W * g[None, :]
    W16 = W.astype(np.float16)
    return (_quant(W16) if int8 else W16.astype(np.float64)), b


# ---- the phase checker -----------------------------------------------------------------------------------------------
class PhaseRun:
    """A forced decode of one model through bstep_kernel, stopped after any grid phase, with its fetched workspace."""

    def __init__(self, m, eng, n, K, n_steps, prompt, seed, int8=False):
        self.m, self.eng, self.n, self.K, self.int8 = m, eng, n, K, int8
        dims = m["dims"]
        self.d, self.H, self.L, self.R = dims.n_text_state, dims.n_text_head, dims.n_text_layer, n * K
        self.n_ctx, self.V = dims.n_text_ctx, dims.n_vocab
        self.vpad = (self.V + 15) // 16 * 16
        self.G = torch.cuda.get_device_properties(0).multi_processor_count
        self.enc = eng.encode(features_for(m, n, seed=seed))
        self.prompts, self.tokens, self.parents = forced_inputs(m["tokens"], n, K, n_steps, seed=seed + 1, prompt=prompt)
        self.P, self.n_steps = len(prompt), n_steps
        self.pos = self.P - 1 + n_steps - 1
        self.w = m["weights"]
        self.slots = np.array([[key_slots(self.P, self.parents, n_steps - 1, b, k, K) for k in range(K)] for b in range(n)])
        self._xkv = None

    def stop(self, p):
        os.environ["B2W_BSTEP_STOP"] = str(p)
        try:
            self.eng.debug_step_logits(self.enc, self.prompts, self.tokens, self.parents)
        finally:
            os.environ.pop("B2W_BSTEP_STOP", None)

    def fetch(self, which, n):
        return self.eng.debug_fetch(which, n).astype(np.float64)

    def x(self):
        nb = (self.d + 127) // 128
        raw = self.eng.debug_fetch(0, nb * self.R * 128).reshape(nb, self.R, 128)
        return raw.transpose(1, 0, 2).reshape(self.R, nb * 128)[:, : self.d].astype(np.float64)

    def raw(self, n_cols):
        parts = self.eng.debug_fetch(1, self.G * self.R * 128).reshape(self.G, self.R, 128)
        return split_k_sum(parts, n_cols, self.d // 64).astype(np.float64)

    def stats(self):
        return ordered_rows_sum(self.eng.debug_fetch(2, (self.d // 64) * self.R * 2).reshape(self.d // 64, self.R, 2)).astype(np.float64)

    def caches(self, l):
        per = self.n * self.n_ctx * self.K * self.d
        shape = (self.L, self.n, self.n_ctx, self.K, self.H, 64)
        kc = self.eng.debug_fetch(9, self.L * per).reshape(shape)[l]
        vc = self.eng.debug_fetch(10, self.L * per).reshape(shape)[l]
        return kc.astype(np.float64), vc.astype(np.float64)

    def xkv(self, l):
        if self._xkv is None:
            per = 2 * self.n * self.H * T_AUDIO * 64
            self._xkv = self.eng.debug_fetch(11, self.L * per).reshape(self.L, 2, self.n, self.H, T_AUDIO, 64)
        return xkv_swizzle(self._xkv[l]).astype(np.float64)

    def fixed(self, raw, s, W, b):
        """The deferred LayerNorm: rstd (raw - mean rowsum W) + b, with mean and rstd from sum x, sum x^2 of the staged tiles."""
        mean = s[:, 0] / self.d
        rstd = 1.0 / np.sqrt(np.maximum(s[:, 1] / self.d - mean * mean, 0) + 1e-5)
        return rstd[:, None] * (raw - mean[:, None] * W.sum(1)[None, :]) + b[None, :]

    def blk(self, l):
        return f"decoder.blocks.{l}"

    def gemm_w(self, l, j):
        p, w, i8 = self.blk(l), self.w, self.int8
        if j == 0:
            return effective(w, [p + ".attn.query.weight", p + ".attn.key.weight", p + ".attn.value.weight"],
                             [p + ".attn.query.bias", p + ".attn.key.bias", p + ".attn.value.bias"], p + ".attn_ln", i8)
        if j == 1:
            return effective(w, [p + ".attn.out.weight"], [p + ".attn.out.bias"], None, i8)
        if j == 2:
            return effective(w, [p + ".cross_attn.query.weight"], [p + ".cross_attn.query.bias"], p + ".cross_attn_ln", i8)
        if j == 3:
            return effective(w, [p + ".cross_attn.out.weight"], [p + ".cross_attn.out.bias"], None, i8)
        if j == 4:
            return effective(w, [p + ".mlp.0.weight"], [p + ".mlp.0.bias"], p + ".mlp_ln", i8)
        return effective(w, [p + ".mlp.2.weight"], [p + ".mlp.2.bias"], None, i8)

    # -- the checks of one phase each; `label` prefixes the printed lines --
    def check_raw(self, label, l, j, x16):
        W, _ = self.gemm_w(l, j)
        raw, want = self.raw(W.shape[0]), x16 @ W.T
        report(label + " raw split-K sums", np.abs(raw - want), ERR_SUM * (np.abs(x16) @ np.abs(W).T) + 1e-6)
        s = self.stats()
        want_s = np.stack([x16.sum(1), (x16 * x16).sum(1)], 1)
        report(label + " row statistics", np.abs(s - want_s), ERR_SUM * np.stack([np.abs(x16).sum(1), (x16 * x16).sum(1)], 1) + 1e-6)

    def check_record(self, label, l, i):
        """The [3L][R][2] statistics record (written by the phase that applies LayerNorm i of layer l) holds what it used."""
        rec = self.fetch(7, 3 * self.L * self.R * 2).reshape(3 * self.L, self.R, 2)[3 * l + i]
        assert np.array_equal(rec, self.stats()), (label, "the statistics record differs from the statistics the phase used")

    def check_resid(self, label, l, j, x_before, a16):
        W, b = self.gemm_w(l, j)
        got, want = self.x() - x_before, a16 @ W.T + b[None, :]
        report(label, np.abs(got - want), ERR_SUM * (np.abs(a16) @ np.abs(W).T + np.abs(x_before)) + 1e-6)

    def self_refs(self, l):
        """q (scaled, fp16 as the kernel holds it), and K, V of every row's visible keys from the fetched cache."""
        W, b = self.gemm_w(l, 0)
        qkv = self.fixed(self.raw(3 * self.d), self.stats(), W, b)
        kc, vc = self.caches(l)
        q16 = (qkv[:, : self.d].astype(np.float16) * np.float16(0.125)).astype(np.float64).reshape(self.n, self.K, self.H, 64)
        Ks = np.empty((self.n, self.K, self.H, self.pos + 1, 64))
        Vs = np.empty_like(Ks)
        j = np.arange(self.pos + 1)
        for bb in range(self.n):
            for k in range(self.K):
                Ks[bb, k] = kc[bb, j, self.slots[bb, k]].transpose(1, 0, 2)
                Vs[bb, k] = vc[bb, j, self.slots[bb, k]].transpose(1, 0, 2)
        return qkv, kc, vc, q16, Ks, Vs

    def check_self(self, label, l, uniform=False):
        qkv, kc, vc, q16, Ks, Vs = self.self_refs(l)
        d, pos = self.d, self.pos
        for name, cache, col in (("k", kc, d), ("v", vc, 2 * d)):
            got = cache[:, pos].reshape(self.R, d)
            want = qkv[:, col:col + d]
            report(label + " %s cache at pos %d" % (name, pos), np.abs(got - want),
                   ERR_LN_REL * np.abs(want).max() + half_ulp(want))
        self.check_record(label, l, 0)
        ao = self.fetch(4, self.R * d).reshape(self.n, self.K, self.H, 64)
        want = attention(q16, Ks, Vs)
        rel = ERR_UNIFORM_REL if uniform else ERR_ATTN_REL
        bound = half_ulp(want) + rel * np.abs(Vs).max() + (0 if uniform else p_rounding_term(q16, Ks, Vs))
        report(label + " attention", np.abs(ao - want), bound)
        if not uniform:
            keys = sorted({0, pos} | set(range(0, pos + 1, 16)))
            check_sensitive(label, lambda j: attention(q16, Ks, Vs, drop=j), keys, bound)

    def check_cross(self, label, l, uniform=False):
        W, b = self.gemm_w(l, 2)
        cq = self.fixed(self.raw(self.d), self.stats(), W, b)
        q16 = (cq.astype(np.float16) * np.float16(0.125)).astype(np.float64).reshape(self.n, self.K, self.H, 64).transpose(0, 2, 1, 3)
        self.check_record(label, l, 1)
        kv = self.xkv(l)
        ao = self.fetch(4, self.R * self.d).reshape(self.n, self.K, self.H, 64).transpose(0, 2, 1, 3)
        want = attention(q16, kv[0][:, :, None], kv[1][:, :, None])
        rel = ERR_UNIFORM_REL if uniform else ERR_ATTN_REL
        bound = half_ulp(want) + rel * np.abs(kv[1]).max() + (0 if uniform else p_rounding_term(q16, kv[0][:, :, None], kv[1][:, :, None]))
        report(label + " attention", np.abs(ao - want), bound)
        if not uniform:
            keys = sorted({0, T_AUDIO - 1} | set(split_starts()))
            check_sensitive(label, lambda j: attention(q16, kv[0][:, :, None], kv[1][:, :, None], drop=j), keys, bound)

    def check_ffn1(self, label, l, x16):
        W, b = self.gemm_w(l, 4)
        s = np.stack([x16.sum(1), (x16 * x16).sum(1)], 1)
        want = gelu(self.fixed(x16 @ W.T, s, W, b))
        got = self.fetch(5, self.R * 4 * self.d).reshape(self.R, 4 * self.d)
        self.check_record(label, l, 2)
        report(label, np.abs(got - want), ERR_LN_REL * np.abs(want).max() + half_ulp(want))


def run_phases(run, only=None, uniform=False):
    """Every grid phase (or those of the kinds in `only`) of `run`, each against float64 on its own fetched inputs."""
    L, d, R = run.L, run.d, run.R
    names = ["qkv", "self", "out", "cross_q", "cross", "cross_out", "ffn1", "ffn2"]
    x_prev = None
    for p in range(1, 3 + 8 * L + 1):
        if 2 <= p <= 1 + 8 * L:
            l, ph = divmod(p - 2, 8)
            kind = names[ph]
        else:
            l, ph, kind = None, None, {1: "embed", 2 + 8 * L: "final_ln"}.get(p, "logits")
        if only is not None and kind not in only:
            continue
        if kind in ("out", "cross_out", "ffn2"):
            run.stop(p - 1)
            x_prev = run.x()
            a16 = run.fetch(5, R * 4 * d).reshape(R, 4 * d) if kind == "ffn2" else run.fetch(4, R * d).reshape(R, d)
        run.stop(p)
        label = "phase %3d %s" % (p, kind if l is None else "L%d %s" % (l, kind))
        if kind == "embed":
            tok = run.tokens[-1].reshape(R)
            want = run.w["decoder.token_embedding.weight"][tok].astype(np.float16).astype(np.float32) + \
                run.w["decoder.positional_embedding"][run.pos].astype(np.float32)
            assert np.array_equal(run.x(), want.astype(np.float64)), label
            print("[decode phases] %-46s bit-exact" % label)
        elif kind in ("qkv", "cross_q"):
            run.check_raw(label, l, 0 if kind == "qkv" else 2, run.x().astype(np.float16).astype(np.float64))
        elif kind == "self":
            run.check_self(label, l, uniform)
        elif kind == "cross":
            run.check_cross(label, l, uniform)
        elif kind in ("out", "cross_out", "ffn2"):
            run.check_resid(label, l, {"out": 1, "cross_out": 3, "ffn2": 5}[kind], x_prev, a16)
        elif kind == "ffn1":
            run.check_raw(label, l, 4, run.x().astype(np.float16).astype(np.float64))
            run.check_ffn1(label + " GELU h16", l, run.x().astype(np.float16).astype(np.float64))
        elif kind == "final_ln":
            x = run.x()
            mean = x.mean(1, keepdims=True)
            want = (x - mean) / np.sqrt(((x - mean) ** 2).mean(1, keepdims=True) + 1e-5)
            got = run.fetch(6, R * d).reshape(R, d)
            report(label, np.abs(got - want), half_ulp(want) + 1e-5 * np.abs(want) + 1e-6)
        else:
            xn = run.fetch(6, R * d).reshape(R, d)
            gf, bf = run.w["decoder.ln.weight"].astype(np.float32), run.w["decoder.ln.bias"].astype(np.float64)
            E = run.w["decoder.token_embedding.weight"].astype(np.float32)
            W16 = (E * gf[None, :]).astype(np.float16)
            W = _quant(W16) if run.int8 else W16.astype(np.float64)
            b = (E.astype(np.float64) @ bf).astype(np.float32).astype(np.float64)
            got = run.fetch(8, R * run.vpad).reshape(R, run.vpad)[:, : run.V]
            report(label, np.abs(got - (xn @ W.T + b[None, :])), ERR_SUM * (np.abs(xn) @ np.abs(W).T) + 1e-4)


# ---- models ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wide():
    """The large-v3 decoder layer (d = 1280, 20 heads, 51866 tokens), 4 decoder layers, as test_gpu_step_logits.py builds it."""
    dims = custom_dims(name="wide", n_mels=128, d=1280, heads=20, enc_layers=1, dec_layers=4, n_vocab=51866)
    return dict(dims=dims, weights=make_weights(dims, seed=13), tokens=special_tokens(dims.n_vocab))


def variant(m, zero_queries=False, pos_offset=0.0):
    """A copy of model m with every decoder query projection (self and cross) zeroed, or a constant added to every channel of the
    decoder's positional embedding."""
    w = dict(m["weights"])
    for l in range(m["dims"].n_text_layer):
        for a in ("attn", "cross_attn"):
            if zero_queries:
                for s in ("weight", "bias"):
                    k = f"decoder.blocks.{l}.{a}.query.{s}"
                    w[k] = np.zeros_like(w[k])
    w["decoder.positional_embedding"] = (w["decoder.positional_embedding"] + np.float32(pos_offset)).astype(np.float32)
    return dict(m, weights=w)


def bstep_engine(m, ct="default"):
    return make_engine(m, compute_type=ct, B2W_STEP="bstep")


PHASE_SHAPES = [(16, 5), (4, 8), (17, 1), (11, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,K", PHASE_SHAPES)
def test_bstep_every_phase(micro_ml, n, K):
    st = micro_ml["tokens"]
    run = PhaseRun(micro_ml, bstep_engine(micro_ml), n, K, 24, prefix_prompt(st), seed=700 + n)
    run_phases(run)


@pytest.mark.gpu
def test_bstep_self_attn_phases_long_context(micro_ml):
    """Prompt [sot] and 447 steps: the last step's rows read every 16-key block and the ancestry table's buffer of an odd position."""
    run = PhaseRun(micro_ml, bstep_engine(micro_ml), 2, 5, 447, [micro_ml["tokens"].sot], seed=720)
    run_phases(run, only={"self"})


@pytest.mark.gpu
@pytest.mark.parametrize("ct", ["default", "int8_float16"])
def test_bstep_every_phase_wide(wide, ct):
    """d = 1280, 20 heads, 16 x 5: 2240 cross-attention tiles in runs of 17 over the CTAs; int8 weights are checked as q x scale."""
    run = PhaseRun(wide, bstep_engine(wide, ct), 16, 5, 6, prefix_prompt(wide["tokens"]), seed=740, int8=ct != "default")
    run_phases(run)


@pytest.mark.gpu
def test_bstep_uniform_queries(micro_ml):
    """Zero queries: each attention phase must return the mean of V over exactly the visible keys."""
    m = variant(micro_ml, zero_queries=True)
    run = PhaseRun(m, bstep_engine(m), 16, 5, 24, prefix_prompt(m["tokens"]), seed=760)
    run_phases(run, only={"self", "cross"}, uniform=True)


@pytest.mark.gpu
@pytest.mark.parametrize("path,n,K", [("dstep", 1, 5), ("dstep", 1, 8), ("layers", 6, 3), ("layers", 1, 9)])
def test_uniform_queries_cross_attention_of_full_steps(micro_ml, path, n, K):
    """Zero queries through dstep_kernel and the layered step: after a full step d_ao holds the last layer's cross-attention output,
    which must be the mean of that layer's cross V over the chunk's 1500 keys."""
    m = variant(micro_ml, zero_queries=True)
    eng = make_engine(m, B2W_STEP=path)
    enc = eng.encode(features_for(m, n, seed=780 + n))
    p, t, par = forced_inputs(m["tokens"], n, K, 8, seed=781, prompt=prefix_prompt(m["tokens"]))
    eng.debug_step_logits(enc, p, t, par)
    dims = m["dims"]
    L, H, d = dims.n_text_layer, dims.n_text_head, dims.n_text_state
    kv = xkv_swizzle(eng.debug_fetch(11, L * 2 * n * H * T_AUDIO * 64).reshape(L, 2, n, H, T_AUDIO, 64)[L - 1]).astype(np.float64)
    got = eng.debug_fetch(4, n * K * d).reshape(n, K, H, 64).astype(np.float64)
    want = kv[1].mean(2)[:, None]
    bound = half_ulp(want) + ERR_UNIFORM_REL * np.abs(kv[1]).max()
    report("uniform %s %dx%d cross-attention" % (path, n, K), np.abs(got - want), bound)
    check_sensitive("uniform %s" % path, lambda j: np.delete(kv[1], j, axis=2).mean(2)[:, None] if j is not None else want,
                    [0, T_AUDIO - 1] + split_starts(), bound)


@pytest.mark.gpu
@pytest.mark.parametrize("offset_sigmas", [8, 32])
def test_bstep_deferred_layernorm_under_a_row_offset(micro_ml, offset_sigmas):
    """A constant added to every channel of the positional embedding shifts the residual rows' mean to about offset_sigmas standard
    deviations.  The K/V cache entries and h16 must stay within the error model of staging the raw residual in fp16."""
    sigma = float(np.std(micro_ml["weights"]["decoder.token_embedding.weight"]))
    m = variant(micro_ml, pos_offset=offset_sigmas * sigma)
    run = PhaseRun(m, bstep_engine(m), 16, 5, 8, prefix_prompt(m["tokens"]), seed=800)
    d, R = run.d, run.R
    for l in range(run.L):
        for j, p in ((0, 3 + 8 * l), (4, 8 + 8 * l)):  # self-attention (k, v written), FFN1 (h16 written)
            run.stop(p)
            x = run.x()
            mean = x.mean(1, keepdims=True)
            rstd = 1.0 / np.sqrt(((x - mean) ** 2).mean(1, keepdims=True) + 1e-5)
            W, b = run.gemm_w(l, j)
            y = ((x - mean) * rstd) @ W.T + b[None, :]
            y16 = (((x - mean) * rstd).astype(np.float16).astype(np.float64)) @ W.T + b[None, :]
            # fp16 staging of x: through W, and through the variance (relative error about 2 u |mean| rstd / sqrt(d)); then the
            # fp16 rounding of the output and fp32 terms
            model = 4 * F16_U * rstd * np.sqrt((x * x) @ (W * W).T) + (2.0 ** -10 + 4 * F16_U * np.abs(mean) * rstd / np.sqrt(d)) * np.abs(y) + 1e-5
            if j == 0:
                kc, vc = run.caches(l)
                got = np.concatenate([kc[:, run.pos].reshape(R, d), vc[:, run.pos].reshape(R, d)], 1)
                y, y16, model = y[:, d:], y16[:, d:], model[:, d:]
            else:
                got = run.fetch(5, R * 4 * d).reshape(R, 4 * d)
                y, y16 = gelu(y), gelu(y16)
            ratio = float(np.abs(mean).mean() * rstd.mean())
            print("[decode phases] offset %d sigma (|mean| / std %.1f) L%d %s: fp16 of the normalised input would give %.3e" % (
                offset_sigmas, ratio, l, "k,v" if j == 0 else "h16", float(np.abs(y16 - y).max())))
            report("offset %d L%d %s" % (offset_sigmas, l, "k,v" if j == 0 else "h16"), np.abs(got - y), model)


# ---- the standalone attention kernels through their hooks ----------------------------------------------------------------
def one_hot_queries(t, K_all):
    """An fp16 query q = gain k_t whose score q k_t / 8 beats every other key's by about 20, and the scores it gives."""
    s0 = K_all @ K_all[t]
    gain = 160.0 / (s0[t] - np.delete(s0, t).max(initial=s0[t] - 20.0))
    q = (gain * K_all[t]).astype(np.float16)
    return q, K_all @ q.astype(np.float64) / 8.0


SELF_H, SELF_CHUNKS, SELF_SLOTS, N_CTX = 2, 2, 16, 448


def self_case(seed, one_hot):
    """448 rows, one per position 0 .. 447, in 2 chunks x 16 slots; both ancestry buffers random over every slot."""
    rng = np.random.default_rng(seed)
    d = 64 * SELF_H
    kc = rng.standard_normal((SELF_CHUNKS, N_CTX, SELF_SLOTS, d)).astype(np.float16)
    vc = rng.standard_normal((SELF_CHUNKS, N_CTX, SELF_SLOTS, d)).astype(np.float16)
    anc = rng.integers(0, SELF_SLOTS, (2, SELF_CHUNKS, SELF_SLOTS, N_CTX)).astype(np.uint8)
    R = N_CTX
    rows = np.array([[i % SELF_CHUNKS, (i * 7) % SELF_SLOTS, i, 0] for i in range(R)], np.int32)
    Ks = np.empty((R, SELF_H, N_CTX, 64))
    Vs = np.empty_like(Ks)
    for r, (b, k, pos, _) in enumerate(rows):
        sl = anc[pos & 1, b, k, : pos + 1].astype(np.int64)
        sl[pos] = k
        Ks[r, :, : pos + 1] = kc[b, np.arange(pos + 1), sl].reshape(pos + 1, SELF_H, 64).transpose(1, 0, 2)
        Vs[r, :, : pos + 1] = vc[b, np.arange(pos + 1), sl].reshape(pos + 1, SELF_H, 64).transpose(1, 0, 2)
    if one_hot:
        tgt = np.array([[(r * 37 + h * 11) % (rows[r, 2] + 1) for h in range(SELF_H)] for r in range(R)])
        q = np.empty((R, SELF_H, 64), np.float16)
        for r in range(R):
            for h in range(SELF_H):
                n = rows[r, 2] + 1
                q[r, h], s = one_hot_queries(tgt[r, h], Ks[r, h, :n])
                assert s[tgt[r, h]] - np.delete(s, tgt[r, h]).max(initial=-np.inf) >= 16
    else:
        tgt = None
        q = (0.5 * rng.standard_normal((R, SELF_H, 64))).astype(np.float16)
    return q, kc, vc, anc, rows, Ks, Vs, tgt


@pytest.mark.gpu
@pytest.mark.parametrize("one_hot", [True, False])
def test_self_attn_kernel(one_hot):
    """dec_self_attn_kernel: every position 0 .. 447, every slot, ancestry pointing at every slot (both buffers)."""
    q, kc, vc, anc, rows, Ks, Vs, tgt = self_case(900 + one_hot, one_hot)
    R = rows.shape[0]
    got = engine.debug_self_attn(q.reshape(R, -1), kc, vc, anc, rows).astype(np.float64).reshape(R, SELF_H, 64)
    if one_hot:
        want = np.stack([[Vs[r, h, tgt[r, h]] for h in range(SELF_H)] for r in range(R)])
        report("self-attn kernel one-hot targets", np.abs(got - want), half_ulp(want) + 1e-4)
        return
    errs, bounds = [], []
    for r in range(R):
        n = rows[r, 2] + 1
        ref = lambda j, r=r, n=n: attention(q[r].astype(np.float64) / 8.0, Ks[r, :, :n], Vs[r, :, :n], drop=j)  # noqa: E731
        want = ref(None)
        bound = half_ulp(want) + ERR_HOOK_REL * np.abs(Vs).max()
        errs.append(np.abs(got[r] - want))
        bounds.append(bound)
        if n > 1:
            check_sensitive("self-attn kernel row %d" % r, ref, sorted({0, n - 1} | set(range(0, n, 16))), bound)
    report("self-attn kernel random", np.stack(errs), np.stack(bounds))


@pytest.mark.gpu
@pytest.mark.parametrize("rpc", [1, 8, 9, 16])
@pytest.mark.parametrize("one_hot", [True, False])
def test_cross_attn_kernel(rpc, one_hot):
    """ds_cross_attn_kernel over 16 chunks x 20 heads: one and two query groups; one-hot targets over every key 0 .. 1499."""
    rng = np.random.default_rng(950 + rpc + 100 * one_hot)
    n, H = 16, 20
    K = rng.standard_normal((n, H, T_AUDIO, 64)).astype(np.float16)
    V = rng.standard_normal((n, H, T_AUDIO, 64)).astype(np.float16)
    K64, V64 = K.astype(np.float64), V.astype(np.float64)
    if one_hot:
        q = np.empty((n, H, rpc, 64), np.float16)
        tgt = (np.arange(n * H * rpc).reshape(n, H, rpc) * 7) % T_AUDIO
        for b in range(n):
            for h in range(H):
                for i in range(rpc):
                    q[b, h, i], s = one_hot_queries(tgt[b, h, i], K64[b, h])
                    assert s[tgt[b, h, i]] - np.delete(s, tgt[b, h, i]).max() >= 16
    else:
        q = (0.5 * rng.standard_normal((n, H, rpc, 64))).astype(np.float16)
    kv = np.stack([xkv_swizzle(K), xkv_swizzle(V)])
    got = engine.debug_cross_attn(q.transpose(0, 2, 1, 3).reshape(n, rpc, H * 64), kv).astype(np.float64)
    got = got.reshape(n, rpc, H, 64).transpose(0, 2, 1, 3)
    if one_hot:
        if rpc == 16:
            assert len(np.unique(tgt)) == T_AUDIO
        want = np.take_along_axis(V64, tgt[..., None], axis=2)
        report("cross-attn kernel one-hot rpc %d" % rpc, np.abs(got - want), half_ulp(want) + 1e-4)
        return
    ref = lambda j: attention(q.astype(np.float64) / 8.0, K64[:, :, None], V64[:, :, None], drop=j)  # noqa: E731
    want = ref(None)
    bound = half_ulp(want) + ERR_HOOK_REL * np.abs(V64).max()
    report("cross-attn kernel random rpc %d" % rpc, np.abs(got - want), bound)
    check_sensitive("cross-attn kernel rpc %d" % rpc, ref, [0, T_AUDIO - 1] + split_starts(), bound)


@pytest.mark.gpu
def test_fetch_rejects_invalid_input(micro_ml):
    m = micro_ml
    eng = bstep_engine(m)
    enc = eng.encode(features_for(m, 2, seed=990))
    p, t, par = forced_inputs(m["tokens"], 2, 5, 2, seed=991, prompt=prefix_prompt(m["tokens"]))
    eng.debug_step_logits(enc, p, t, par)
    L, d = m["dims"].n_text_layer, m["dims"].n_text_state
    eng.debug_fetch(9, L * 2 * m["dims"].n_text_ctx * 5 * d)  # the valid call runs
    for which, n in ((3, 1), (12, 1), (4, 80 * d + 1), (9, L * 2 * m["dims"].n_text_ctx * 5 * d + L), (10, L + 1),
                     (11, L * 2 * 2 * 1500 * d + 1)):
        with pytest.raises(ValueError):
            eng.debug_fetch(which, n)


# ---- CPU: the helpers on hand-worked cases ---------------------------------------------------------------------------------
def test_key_slots_hand_worked():
    """Prompt of 2 (one prefilled key, in slot 0), 3 slots, 3 steps.  Step 1: slot 0 continues slot 2, slots 1 and 2 continue
    slot 0.  Step 2: slots 0 and 1 continue slot 1, slot 2 continues itself."""
    parents = np.zeros((3, 1, 3), np.int32)
    parents[1, 0] = [2, 0, 0]
    parents[2, 0] = [1, 1, 2]
    # row 0 at step 2 continues slot 1 (step 1), which continued slot 0 (step 0)
    assert key_slots(2, parents, 2, 0, 0, 3).tolist() == [0, 0, 1, 0]
    assert key_slots(2, parents, 2, 0, 1, 3).tolist() == [0, 0, 1, 1]
    assert key_slots(2, parents, 2, 0, 2, 3).tolist() == [0, 0, 2, 2]
    assert key_slots(2, parents, 1, 0, 0, 3).tolist() == [0, 2, 0]
    assert key_slots(1, None, 2, 0, 2, 3).tolist() == [2, 2, 2]


def test_xkv_swizzle_hand_worked():
    T = 9
    x = (np.arange(T)[:, None] * 64 + np.arange(64)[None, :]).astype(np.float32)
    y = xkv_swizzle(x)
    assert y[0].tolist() == x[0].tolist()
    # key 3: stored chunk c holds chunk c ^ 3, so stored chunk 0 holds elements 24..31
    assert y[3, 0:8].tolist() == (3 * 64 + np.arange(24, 32)).tolist()
    assert y[3, 24:32].tolist() == (3 * 64 + np.arange(0, 8)).tolist()
    assert y[8].tolist() == x[8].tolist()  # 8 & 7 = 0
    assert np.array_equal(xkv_swizzle(y), x)


def test_split_k_sum_order_hand_worked():
    """7 CTAs, 2 n-blocks of 3 k-atoms: n-block 0 is CTAs 0-2, n-block 1 CTAs 4-6 (CTA 3 has no atom).  Summed in CTA order,
    1e8 + (-1e8) + 1 is 1 in fp32; any other order loses the 1."""
    parts = np.zeros((7, 1, 128), np.float32)
    parts[0, 0, :], parts[1, 0, :], parts[2, 0, :] = 1e8, -1e8, 1.0
    parts[3] = np.nan
    parts[4, 0, :], parts[5, 0, :], parts[6, 0, :] = 2.0, 3.0, 4.0
    assert bs_group(2, 3, 7, 0) == (0, 3) and bs_group(2, 3, 7, 1) == (4, 3)
    out = split_k_sum(parts, 200, 3)
    assert out.shape == (1, 200)
    assert (out[0, :128] == 1.0).all() and (out[0, 128:] == 9.0).all()
    st = np.array([[[1e8, 0.0]], [[-1e8, 1.0]], [[1.0, 2.0]]], np.float32)
    assert ordered_rows_sum(st).tolist() == [[1.0, 3.0]]


def test_attention_reference_and_sensitivity_helpers():
    rng = np.random.default_rng(3)
    K, V = rng.standard_normal((5, 64)), rng.standard_normal((5, 64))
    q = np.zeros(64)
    assert np.allclose(attention(q, K, V), V.mean(0))
    assert np.allclose(attention(q, K, V, drop=2), np.delete(V, 2, 0).mean(0))
    check_sensitive("mean of 5", lambda j: attention(q, K, V, drop=j), [0, 4], 1e-3)
    with pytest.raises(AssertionError):
        check_sensitive("mean of 5", lambda j: attention(q, K, V, drop=j), [0], 10.0)
