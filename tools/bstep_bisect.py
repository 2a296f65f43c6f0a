"""Phase-by-phase check of the many-row persistent step kernel (csrc/bstep.cu) on a GPU box.

Runs ONE decode step (prompt [sot, notimestamps], so the step feeds position 1 after a one-token prefill) with
B2W_STEP=bstep and B2W_BSTEP_STOP=p for p = 1 .. number of grid phases, fetches the decoder workspace after each
stop (b2w_debug_fetch) and compares it with a NumPy restatement of the same step.  Prints the max abs error per
phase so one run bisects a wrong kernel.  The QKV and cross-q outputs exist only as the CTAs' split-K partial tiles and
per-k-atom row statistics (their consumers sum them): those are summed here in the kernel's order.  Test infrastructure (imports oracle/ only for the log-mel features).

    python tools/bstep_bisect.py [--chunks 2] [--beam 5] [--d 128] [--layers 2]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def ln(x, eps=1e-5):
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps)


def gelu(x):
    from math import erf

    return 0.5 * x * (1.0 + np.vectorize(erf)(x / np.sqrt(2.0)))


def softmax(s):
    s = s - s.max(-1, keepdims=True)
    e = np.exp(s)
    return e / e.sum(-1, keepdims=True)


def reference_step(w, enc, toks, d, H, L):
    """Teacher-forced decoder over `toks` (positions 0..n-1) for one chunk; returns per-phase values of the LAST position."""
    n = len(toks)
    x = w["decoder.token_embedding.weight"][toks] + w["decoder.positional_embedding"][:n]
    out = {}
    mask = np.triu(np.full((n, n), -np.inf), 1)
    for l in range(L):
        p = f"decoder.blocks.{l}"
        g, b = w[p + ".attn_ln.weight"], w[p + ".attn_ln.bias"]
        xn = ln(x) * g + b
        q = xn @ w[p + ".attn.query.weight"].T + w[p + ".attn.query.bias"]
        k = xn @ w[p + ".attn.key.weight"].T
        v = xn @ w[p + ".attn.value.weight"].T + w[p + ".attn.value.bias"]
        out[(l, 0)] = np.concatenate([q[-1], k[-1], v[-1]])
        ao = np.zeros_like(q)
        for h in range(H):
            sl = slice(64 * h, 64 * h + 64)
            s = q[:, sl] @ k[:, sl].T / 8.0 + mask
            ao[:, sl] = softmax(s) @ v[:, sl]
        out[(l, 1)] = ao[-1]
        x = x + ao @ w[p + ".attn.out.weight"].T + w[p + ".attn.out.bias"]
        out[(l, 2)] = x[-1].copy()
        g, b = w[p + ".cross_attn_ln.weight"], w[p + ".cross_attn_ln.bias"]
        xn = ln(x) * g + b
        cq = xn @ w[p + ".cross_attn.query.weight"].T + w[p + ".cross_attn.query.bias"]
        out[(l, 3)] = cq[-1]
        ck = enc @ w[p + ".cross_attn.key.weight"].T
        cv = enc @ w[p + ".cross_attn.value.weight"].T + w[p + ".cross_attn.value.bias"]
        ao = np.zeros_like(cq)
        for h in range(H):
            sl = slice(64 * h, 64 * h + 64)
            ao[:, sl] = softmax(cq[:, sl] @ ck[:, sl].T / 8.0) @ cv[:, sl]
        out[(l, 4)] = ao[-1]
        x = x + ao @ w[p + ".cross_attn.out.weight"].T + w[p + ".cross_attn.out.bias"]
        out[(l, 5)] = x[-1].copy()
        g, b = w[p + ".mlp_ln.weight"], w[p + ".mlp_ln.bias"]
        xn = ln(x) * g + b
        hpre = xn @ w[p + ".mlp.0.weight"].T + w[p + ".mlp.0.bias"]
        out[(l, 6)] = hpre[-1]
        hh = gelu(hpre)
        out[(l, 7)] = hh[-1]
        x = x + hh @ w[p + ".mlp.2.weight"].T + w[p + ".mlp.2.bias"]
        out[(l, 8)] = x[-1].copy()
    out["xn"] = ln(x)[-1]
    xf = ln(x) * w["decoder.ln.weight"] + w["decoder.ln.bias"]
    out["logits"] = (xf @ w["decoder.token_embedding.weight"].T)[-1]
    out["embed"] = (w["decoder.token_embedding.weight"][toks] + w["decoder.positional_embedding"][:n])[-1]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=2)
    ap.add_argument("--beam", type=int, default=5)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--first", type=int, default=1)
    ap.add_argument("--last", type=int, default=0)
    args = ap.parse_args()
    os.environ["B2W_STEP"] = "bstep"
    from faster_whisper_b200 import engine
    from faster_whisper_b200.config import special_tokens
    from faster_whisper_b200.synthetic import custom_dims, make_weights, synthetic_audio
    from oracle.whisper_oracle import log_mel, pad_or_trim

    d, L, B, K = args.d, args.layers, args.chunks, args.beam
    H = d // 64
    dims = custom_dims(d=d, heads=H, enc_layers=1, dec_layers=L, n_vocab=51864)
    w = make_weights(dims, seed=3)
    st = special_tokens(dims.n_vocab)
    eng = engine.Whisper(dims=dims, weights=w, tokens=st, device="cuda")
    feats = np.stack([pad_or_trim(log_mel(synthetic_audio(70 + i, 30.0), dims.n_mels)[:, :-1]) for i in range(B)])
    enc = eng.encode(feats)
    enc_np = enc.numpy().astype(np.float64)
    w64 = {k: v.astype(np.float64) for k, v in w.items() if k.startswith("decoder.")}
    toks = [st.sot, st.no_timestamps]
    refs = [reference_step(w64, enc_np[b], toks, d, H, L) for b in range(B)]
    R = B * K
    vpad = (dims.n_vocab + 15) // 16 * 16
    nph = 3 + 8 * L
    import torch

    G = torch.cuda.get_device_properties(0).multi_processor_count  # the step kernel's grid: one CTA per SM
    KA = d // 64
    last = args.last or nph

    def rows(key):
        return np.stack([refs[r // K][key] for r in range(R)])

    def fetch_blocked(which, n_cols):
        """fp32 accumulate buffers are n-block-major: [(n >> 7)][row][n & 127]."""
        nb = (n_cols + 127) // 128
        raw = eng.debug_fetch(which, nb * R * 128).reshape(nb, R, 128)
        return raw.transpose(1, 0, 2).reshape(R, nb * 128)[:, :n_cols]

    def split_k_sum(n_cols):
        """GEMM output [R][n_cols] from the partial tiles [CTA][R][128]: n-block nb is summed over its CTAs g0 .. g0 + gn - 1 in
        CTA order, fp32 (bs_group in csrc/bstep.cu)."""
        NB = (n_cols + 127) // 128
        parts = eng.debug_fetch(1, G * R * 128).reshape(G, R, 128)
        base, extra = G // NB, G % NB
        out = np.zeros((R, NB * 128), np.float32)
        for nb in range(NB):
            g0, gn = nb * base + min(nb, extra), min(base + 1 if nb < extra else base, KA)
            t = parts[g0].copy()
            for k in range(1, gn):
                t = t + parts[g0 + k]
            out[:, nb * 128 : nb * 128 + 128] = t
        return out[:, :n_cols]

    def row_stats():
        """sum(x), sum(x^2) per row: the per-k-atom partials [KA][R][2] summed in k order, fp32."""
        stp = eng.debug_fetch(2, KA * R * 2).reshape(KA, R, 2)
        t = stp[0].copy()
        for k in range(1, KA):
            t = t + stp[k]
        return t.astype(np.float64)

    def fixed(raw, lname, wname, bname, s):
        p_ln_g, p_ln_b = w64[lname + ".weight"], w64[lname + ".bias"]
        Ws = w64[wname] if isinstance(wname, str) else np.concatenate([w64[x] for x in wname])
        bs = np.concatenate([w64[x] if x in w64 else np.zeros(d) for x in bname]) if not isinstance(bname, str) else w64[bname]
        Wf = (Ws * p_ln_g[None, :]).astype(np.float16).astype(np.float64)
        bf = bs + Ws @ p_ln_b
        mean = s[:, 0] / d
        rstd = 1.0 / np.sqrt(np.maximum(s[:, 1] / d - mean * mean, 0) + 1e-5)
        return rstd[:, None] * (raw - mean[:, None] * Wf.sum(1)[None, :]) + bf[None, :]

    names = ["qkv", "self", "out", "cross_q", "cross", "cross_out", "ffn1+gelu", "ffn2"]
    ref_key = [0, 1, 2, 3, 4, 5, 7, 8]  # reference_step's value after each grid phase of a layer
    worst = 0.0
    for p in range(args.first, last + 1):
        os.environ["B2W_BSTEP_STOP"] = str(p)
        eng.generate(enc, [toks] * B, beam_size=K, max_length=len(toks) + 1, return_scores=True)
        if p == 1:
            got, want, label = fetch_blocked(0, d), rows("embed"), "embed x"
        elif p <= 1 + 8 * L:
            l, ph = divmod(p - 2, 8)
            blk = f"decoder.blocks.{l}"
            label = f"L{l} {names[ph]}"
            want = rows((l, ref_key[ph]))
            if ph == 0:
                raw = split_k_sum(3 * d).astype(np.float64)
                got = fixed(raw, blk + ".attn_ln", [blk + ".attn.query.weight", blk + ".attn.key.weight", blk + ".attn.value.weight"],
                            [blk + ".attn.query.bias", blk + ".attn.key.bias", blk + ".attn.value.bias"], row_stats())
            elif ph in (1, 4):
                got = eng.debug_fetch(4, R * d).reshape(R, d)
            elif ph in (2, 5, 7):
                got = fetch_blocked(0, d)
            elif ph == 3:
                raw = split_k_sum(d).astype(np.float64)
                got = fixed(raw, blk + ".cross_attn_ln", blk + ".cross_attn.query.weight", blk + ".cross_attn.query.bias", row_stats())
            else:
                got = eng.debug_fetch(5, R * 4 * d).reshape(R, 4 * d)
        elif p == 2 + 8 * L:
            got, want, label = eng.debug_fetch(6, R * d).reshape(R, d), rows("xn"), "final LN"
        else:
            got, want, label = eng.debug_fetch(8, R * vpad).reshape(R, vpad)[:, : dims.n_vocab], rows("logits"), "logits"
        err = np.abs(np.asarray(got, np.float64) - want)
        bad = int(np.argmax(err.max(1)))
        print("phase %3d %-14s max abs err %.4g (ref max %.3g) worst row %d col %d nan %d" % (
            p, label, err.max(), np.abs(want).max(), bad, int(np.argmax(err[bad])), int(np.isnan(np.asarray(got)).sum())), flush=True)
        worst = max(worst, float(err.max()) if np.isfinite(err.max()) else 1e9)
    os.environ.pop("B2W_BSTEP_STOP", None)
    print("worst", worst, flush=True)
    return 0 if worst < 0.08 else 1


if __name__ == "__main__":
    sys.exit(main())
