"""-m gpu: the dense wgmma GEMM and the decoder's GEMM route against float64 NumPy, at the shapes, epilogues and schedules the
engine runs; the encoder's batch invariance; the flash attention's rescaling.

Operands are fp16-rounded and the reference is float64 on them.  Bounds (largest values measured on an H100 80GB HBM3 at 700 W
in the comments): fp32 outputs |got - want| <= TOL * max(1, |want|); fp16 outputs one fp16 ulp of want plus that, against want rounded
to fp16.  Every output buffer starts filled with a NaN sentinel no kernel computes: elements outside the valid set (padding rows
and columns, a guard after the buffer, cache entries no row addresses) must keep it, and every valid element must have been
written.
"""
import functools
import math

import numpy as np
import pytest
from scipy.special import erf

from faster_whisper_b200 import engine
from faster_whisper_b200.engine import (EPI_F16, EPI_F16_XKV, EPI_F32, EPI_GELU_F16, EPI_GELU_POS_F32, EPI_QKV_CACHE, EPI_RESID_F32,
                                        GV_F16, GV_F32, GV_GELU_F16, GV_QKV, GV_RESID_LN)

pytestmark = pytest.mark.gpu

TOL_GEMM = 2e-5  # dense GEMM and conv stem; measured 5.4e-6 (conv2), fp16 outputs 1.9e-6 beyond one ulp
TOL_GV = 6e-5  # decoder GEMM, both routes; measured 2.5e-5 (LayerNorm after the wgmma residual update, d = 1280), 8.5e-6 fp32
TOL_ATTN = 2e-3  # flash attention with a late maximum, absolute (fp16 probabilities and output); measured 7.1e-4
GUARD = 1024  # elements after the last one a kernel may write
SENT16 = np.uint16(0x7E5A)
SENT32 = np.uint32(0x7FC0BEEF)
VPAD = 51872  # large-v3's padded vocabulary: the logits GEMM's N


def sentinel(shape, dtype):
    a = np.empty(shape, dtype)
    a.view(np.uint16 if dtype == np.float16 else np.uint32)[...] = SENT16 if dtype == np.float16 else SENT32
    return a


def untouched(a):
    return a.view(np.uint16) == SENT16 if a.dtype == np.float16 else a.view(np.uint32) == SENT32


def r16(rng, shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float16)


def gelu(x):
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


def check(name, got, want, tol, quiet=False):
    """got (float32 or float16) against float64 want; fp16 outputs are compared with want rounded to fp16, plus one ulp."""
    want = np.asarray(want, np.float64)
    scale = np.maximum(1.0, np.abs(want))
    if got.dtype == np.float16:
        w16 = want.astype(np.float16)
        err = np.abs(got.astype(np.float64) - w16.astype(np.float64))
        ulp = np.spacing(np.abs(w16)).astype(np.float64)
        excess = np.maximum(err - ulp, 0.0) / scale
    else:
        err = np.abs(got.astype(np.float64) - want)
        excess = err / scale
    assert got.shape == want.shape, (name, got.shape, want.shape)
    assert np.isfinite(got).all(), f"{name}: {int((~np.isfinite(got)).sum())} elements not written or not finite"
    worst = float(excess.max()) if excess.size else 0.0
    if not quiet:
        print(f"[measured] {name}: max |err| {float(err.max()):.3g}, max error / bound scale {worst:.3g} (bound {tol:g})")
    assert worst <= tol, (name, worst, np.unravel_index(int(excess.argmax()), excess.shape))
    return worst


# ---- dense GEMM ----------------------------------------------------------------------------------------------------
F16_OUT = (EPI_F16, EPI_GELU_F16, EPI_F16_XKV, EPI_QKV_CACHE)
EPI_NAMES = {EPI_F16: "f16", EPI_GELU_F16: "gelu_f16", EPI_RESID_F32: "resid_f32", EPI_GELU_POS_F32: "gelu_pos_f32",
             EPI_F32: "f32", EPI_F16_XKV: "f16_xkv", EPI_QKV_CACHE: "qkv_cache"}
# N per epilogue: 192 and 576 are not multiples of 128 (partial last 128-wide tile); XKV is 3 layers x K,V x 3 heads
EPI_N = {EPI_F16: 576, EPI_GELU_F16: 192, EPI_RESID_F32: 192, EPI_GELU_POS_F32: 576, EPI_F32: 192, EPI_F16_XKV: 1152, EPI_QKV_CACHE: 576}


class GemmCase:
    """Inputs, the float64 reference and the sentinel-filled outputs of one dense GEMM shaped as the engine states it.
    bn 128: 1500 rows per batch item (the last M tile is partial); bn 32: 80 rows, one M tile, narrow tiles."""

    def __init__(self, epi, bn, a_batch, N=None, K=None, rows=None, seed=0):
        rng = np.random.default_rng(seed * 1000 + epi * 10 + bn + a_batch)
        self.epi, self.bn, self.B = epi, bn, a_batch
        N = N or EPI_N[epi]
        K = K or (448 if bn == 128 else 576)  # more 64-wide K blocks than the ring has stages
        rows = rows or (1500 if bn == 128 else 80)
        self.N, self.K, self.rows = N, K, rows
        # A with padding columns and rows between batch items that must never be read (large values would show)
        lda, a_rows = K + 64, rows
        a_bstride = (rows + 7) * lda
        a = np.full((a_batch * a_bstride,), 1000.0, np.float16)
        av = r16(rng, (a_batch, rows, K))
        for b in range(a_batch):
            a[b * a_bstride:b * a_bstride + rows * lda].reshape(rows, lda)[:, :K] = av[b]
        w = r16(rng, (N, K), 1.0 / math.sqrt(K))
        bias = rng.standard_normal(N).astype(np.float32)
        y = np.einsum("brk,nk->brn", av.astype(np.float64), w.astype(np.float64)) + bias
        self.kw = dict(epilogue=epi, rows=rows, a_batch=a_batch, a_rows=a_rows, a_cols=K, a_row_stride=lda, a_batch_stride=a_bstride,
                       bias=bias, narrow_tiles=bn == 32)
        self.a, self.w = a, w
        dt = np.float16 if epi in F16_OUT else np.float32
        self.kcache = self.vcache = None
        if epi == EPI_F16_XKV:
            L, H, T = N // 384, 3, rows + (16 if bn == 32 else 0)
            self.xkv = (L, H, T)
            self.out = sentinel(N * a_batch * T + GUARD, np.float16)
            self.kw.update(xkv=(64 * H, H, T, a_batch))
            self.want = y
        elif epi == EPI_QKV_CACHE:
            d, n_ctx, slots, chunks = N // 3, 448, 16, 2
            flat = rng.choice(chunks * n_ctx * slots, rows, replace=False)  # distinct (chunk, pos, slot)
            chunk, rem = np.divmod(flat, n_ctx * slots)
            pos, slot = np.divmod(rem, slots)
            self.rowinfo = np.stack([chunk, slot, pos, np.zeros_like(pos)], 1).astype(np.int32)
            self.out = sentinel(rows * d + GUARD, np.float16)
            self.kcache = sentinel((chunks, n_ctx, slots, d), np.float16)
            self.vcache = sentinel((chunks, n_ctx, slots, d), np.float16)
            self.kw.update(rowinfo=self.rowinfo, qkv_d=d, n_ctx=n_ctx, slots=slots)
            self.want = y[0]
        else:
            ld, ob = N + 32, (rows + 5) * (N + 32)
            self.out = sentinel(a_batch * ob + GUARD, dt)
            self.kw.update(out_ld=ld, out_batch_stride=ob)
            if epi == EPI_RESID_F32:
                resid = rng.standard_normal((a_batch, rows, N)).astype(np.float32)
                self.view(self.out)[...] = resid
                y = y + resid
            elif epi == EPI_GELU_POS_F32:
                pos = rng.standard_normal((rows, N)).astype(np.float32)
                self.kw.update(pos=pos)
                y = gelu(y) + pos
            elif epi == EPI_GELU_F16:
                y = gelu(y)
            self.want = y

    def view(self, out):
        """The valid [B][rows][N] region of a strided output."""
        ld, ob = self.kw["out_ld"], self.kw["out_batch_stride"]
        return np.lib.stride_tricks.as_strided(out, (self.B, self.rows, self.N),
                                               (ob * out.itemsize, ld * out.itemsize, out.itemsize), writeable=True)

    def run(self, max_ctas=0, impl=0):
        out = self.out.copy()
        kc = None if self.kcache is None else self.kcache.copy()
        vc = None if self.vcache is None else self.vcache.copy()
        bn, grid = engine.debug_gemm_desc(self.a, self.w, out, kcache=kc, vcache=vc, max_ctas=max_ctas, impl=impl, **self.kw)
        if impl == 0:
            assert bn == self.bn, (bn, self.bn)
        return out, kc, vc, grid

    def check(self, out, kc, vc, name):
        epi, B, rows, N = self.epi, self.B, self.rows, self.N
        if epi == EPI_F16_XKV:
            L, H, T = self.xkv
            body = out[:N * B * T].reshape(L, 2, B, H, T, 8, 8)
            t = np.arange(T)
            got = body[:, :, :, :, t[:, None], np.arange(8)[None, :] ^ (t[:, None] & 7), :].reshape(L, 2, B, H, T, 64)
            want = self.want.reshape(B, rows, L, 2, H, 64).transpose(2, 3, 0, 4, 1, 5)
            check(name, got[:, :, :, :, :rows], want, TOL_GEMM)
            assert untouched(got[:, :, :, :, rows:]).all(), "XKV positions past the rows were written"
            assert untouched(out[N * B * T:]).all(), "guard after the XKV buffer was written"
        elif epi == EPI_QKV_CACHE:
            d = N // 3
            check(name + " q", out[:rows * d].reshape(rows, d), self.want[:, :d], TOL_GEMM)
            assert untouched(out[rows * d:]).all(), "guard after q was written"
            c, s, p = self.rowinfo[:, 0], self.rowinfo[:, 1], self.rowinfo[:, 2]
            check(name + " k", kc[c, p, s], self.want[:, d:2 * d], TOL_GEMM)
            check(name + " v", vc[c, p, s], self.want[:, 2 * d:], TOL_GEMM)
            for cache in (kc, vc):
                hit = np.zeros(cache.shape[:3], bool)
                hit[c, p, s] = True
                assert untouched(cache[~hit]).all(), "a cache entry no row addresses was written"
        else:
            check(name, self.view(out), self.want, TOL_GEMM)
            mask = np.ones(out.shape, bool)
            self.view(mask)[...] = False
            assert untouched(out[mask]).all(), "padding rows / columns or the guard were written"


EPI_CASES = [(e, 128, b) for e in EPI_NAMES for b in (1, 3) if not (e == EPI_QKV_CACHE and b == 3)] + [(e, 32, 1) for e in EPI_NAMES]


@pytest.mark.parametrize("epi,bn,a_batch", EPI_CASES, ids=[f"{EPI_NAMES[e]}-bn{bn}-b{b}" for e, bn, b in EPI_CASES])
def test_gemm_epilogue(epi, bn, a_batch):
    c = GemmCase(epi, bn, a_batch)
    out, kc, vc, _ = c.run()
    c.check(out, kc, vc, f"gemm {EPI_NAMES[epi]} bn{bn} b{a_batch}")


def test_gemm_logits_shape():
    """N = 51 872 (large-v3's padded vocabulary) at 80 rows: too many 128-wide tiles for narrow ones, partial last tile."""
    c = GemmCase(EPI_F32, 128, 1, N=VPAD, K=192, rows=80)
    c.kw["narrow_tiles"] = True
    out, kc, vc, _ = c.run()
    c.check(out, kc, vc, "gemm logits")


@pytest.mark.parametrize("epi", [EPI_F32, EPI_QKV_CACHE, EPI_F16_XKV])
def test_gemm_simt_reference_same_contract(epi):
    """The SIMT reference GEMM (the engine's bisecting path) meets the same contract."""
    c = GemmCase(epi, 128, 1 if epi == EPI_QKV_CACHE else 3)
    out, kc, vc, _ = c.run(impl=1)
    c.check(out, kc, vc, f"gemm simt {EPI_NAMES[epi]}")


# ---- conv stem: implicit GEMM over taps ----------------------------------------------------------------------------------
def conv1d_ref(x, w, stride):
    """float64 conv1d(padding=1): x [B][T][Cin], w [Cout][Cin][3] -> [B][T_out][Cout]."""
    B, T, _ = x.shape
    xp = np.zeros((B, T + 2, x.shape[2]))
    xp[:, 1:-1] = x
    To = T // stride
    return sum(xp[:, k:k + stride * To:stride] @ w[:, :, k].T.astype(np.float64) for k in range(3))


def conv_cases(n_mels, seed=0):
    """conv1 (3 row taps over channel-padded features, GELU, fp16) and conv2 (stride 2 as a row-pair view, GELU + pos, fp32)
    for 3 chunks at d = 192, packed as encoder_plan packs them."""
    rng = np.random.default_rng(seed + n_mels)
    B, d, cpad = 3, 192, 128
    feats = r16(rng, (B, 3000, n_mels))
    x0 = np.zeros((B, 3000, cpad), np.float16)
    x0[:, :, :n_mels] = feats
    w1 = r16(rng, (d, n_mels, 3), 1.0 / math.sqrt(3 * n_mels))
    W1 = np.zeros((d, 3, cpad), np.float16)
    W1[:, :, :n_mels] = w1.transpose(0, 2, 1)
    b1 = rng.standard_normal(d).astype(np.float32)
    want1 = gelu(conv1d_ref(feats.astype(np.float64), w1, 1) + b1)
    conv1 = dict(a=x0.reshape(-1), w=W1.reshape(d, 3 * cpad), want=want1, shape=(B, 3000, d),
                 kw=dict(epilogue=EPI_GELU_F16, rows=3000, a_batch=B, a_rows=3000, a_cols=cpad, a_batch_stride=3000 * cpad,
                         tap_row=(-1, 0, 1), tap_col=(0, 0, 0), bias=b1, out_ld=d, out_batch_stride=3000 * d))
    x1 = r16(rng, (B, 3000, d))
    w2 = r16(rng, (d, d, 3), 1.0 / math.sqrt(3 * d))
    b2 = rng.standard_normal(d).astype(np.float32)
    pos = rng.standard_normal((1500, d)).astype(np.float32)
    want2 = gelu(conv1d_ref(x1.astype(np.float64), w2, 2) + b2) + pos
    conv2 = dict(a=x1.reshape(-1), w=np.ascontiguousarray(w2.transpose(0, 2, 1).reshape(d, 3 * d)), want=want2, shape=(B, 1500, d),
                 kw=dict(epilogue=EPI_GELU_POS_F32, rows=1500, a_batch=B, a_rows=1500, a_cols=2 * d, a_batch_stride=3000 * d,
                         tap_row=(-1, 0, 0), tap_col=(d, 0, d), bias=b2, pos=pos, out_ld=d, out_batch_stride=1500 * d))
    return conv1, conv2


def run_conv(c, max_ctas=0):
    n = int(np.prod(c["shape"]))
    out = sentinel(n + GUARD, np.float16 if c["kw"]["epilogue"] == EPI_GELU_F16 else np.float32)
    engine.debug_gemm_desc(c["a"], c["w"], out, max_ctas=max_ctas, **c["kw"])
    return out


@pytest.mark.parametrize("n_mels", [80, 128])
def test_conv_stem_is_a_convolution(n_mels):
    for name, c in zip(("conv1", "conv2"), conv_cases(n_mels)):
        out = run_conv(c)
        n = int(np.prod(c["shape"]))
        got = out[:n].reshape(c["shape"])
        # the first and last output rows read a tap outside the chunk, which must load as zeros
        check(f"{name} n_mels={n_mels} t=0", got[:, 0], c["want"][:, 0], TOL_GEMM)
        check(f"{name} n_mels={n_mels} t=last", got[:, -1], c["want"][:, -1], TOL_GEMM)
        check(f"{name} n_mels={n_mels}", got, c["want"], TOL_GEMM)
        assert untouched(out[n:]).all()


# ---- persistent schedule: several tiles per CTA ---------------------------------------------------------------------------
SCHED_CASES = [(e, 128, 1 if e == EPI_QKV_CACHE else 3) for e in EPI_NAMES] + [(e, 32, 1) for e in EPI_NAMES]


@pytest.mark.parametrize("epi,bn,a_batch", SCHED_CASES, ids=[f"{EPI_NAMES[e]}-bn{bn}-b{b}" for e, bn, b in SCHED_CASES])
def test_gemm_persistent_schedule_bit_identical(epi, bn, a_batch):
    """Each output element belongs to one tile with a fixed K order, so 1, 3 or 7 CTAs walking all tiles (tile counts that are
    not multiples of the grid) give exactly the bits of one CTA per SM."""
    c = GemmCase(epi, bn, a_batch, seed=1)
    base = c.run()
    assert base[3] > 3
    for max_ctas in (1, 3, 7):
        got = c.run(max_ctas=max_ctas)
        assert got[3] == min(max_ctas, base[3])
        for g, b in zip(got[:3], base[:3]):
            if b is not None:
                assert np.array_equal(g.view(np.uint8), b.view(np.uint8)), f"max_ctas={max_ctas} changed the result"


@pytest.mark.parametrize("conv", ["conv1", "conv2"])
def test_conv_stem_persistent_schedule_bit_identical(conv):
    c = conv_cases(80, seed=3)[conv == "conv2"]
    base = run_conv(c)
    for max_ctas in (1, 3, 7):
        assert np.array_equal(run_conv(c, max_ctas).view(np.uint8), base.view(np.uint8)), max_ctas


# ---- the decoder's GEMM route, 1..80 rows ------------------------------------------------------------------------------------
GV_NAMES = {GV_QKV: "qkv", GV_F16: "f16", GV_GELU_F16: "gelu_f16", GV_RESID_LN: "resid_ln", GV_F32: "f32"}


@functools.lru_cache(maxsize=None)
def gv_inputs(mode, d):
    """80 rows of inputs and their float64 results: the first R rows are the R-row case."""
    rng = np.random.default_rng((mode if mode in GV_NAMES else 9) * 7 + d)
    N, K = {GV_QKV: (3 * d, d), GV_F16: (d, d), GV_GELU_F16: (4 * d, d), GV_RESID_LN: (d, 4 * d), GV_F32: (d, d)}.get(mode, (VPAD, d))
    if mode == "logits":
        mode = GV_F32
    x = r16(rng, (80, K))
    w = r16(rng, (N, K), 1.0 / math.sqrt(K))
    bias = rng.standard_normal(N).astype(np.float32)
    y = x.astype(np.float64) @ w.astype(np.float64).T + bias
    inp = dict(mode=mode, x=x, w=w, bias=bias, N=N, K=K, y=y)
    if mode == GV_QKV:
        n_ctx, slots = 448, 8
        flat = rng.choice(n_ctx * slots, 80, replace=False)
        pos, slot = np.divmod(flat, slots)
        inp["rows"] = np.stack([np.zeros_like(pos), slot, pos, np.zeros_like(pos)], 1).astype(np.int32)
        inp["cache"] = (1, n_ctx, slots, d)
    if mode == GV_GELU_F16:
        inp["y"] = gelu(y)
    if mode == GV_RESID_LN:
        xres = rng.standard_normal((80, N)).astype(np.float32)
        g = (1.0 + 0.5 * rng.standard_normal(N)).astype(np.float32)
        b = rng.standard_normal(N).astype(np.float32)
        xnew = xres + y
        mean = xnew.mean(1, keepdims=True)
        var = ((xnew - mean) ** 2).mean(1, keepdims=True)
        inp.update(xres=xres, ln_g=g, ln_b=b, y=xnew, xn=(xnew - mean) / np.sqrt(var + 1e-5) * g + b)
    return inp


def run_gv(inp, R, route):
    mode, N, d = inp["mode"], inp["N"], inp["N"] // 3
    kw = dict(mode=mode, bias=inp["bias"], route=route)
    res = {}
    if mode == GV_QKV:
        kc, vc = sentinel(inp["cache"], np.float16), sentinel(inp["cache"], np.float16)
        out = sentinel(R * d + GUARD, np.float16)
        kw.update(out=out, rows=inp["rows"][:R], kcache=kc, vcache=vc, d=d, n_ctx=inp["cache"][1], slots=inp["cache"][2])
        res.update(kc=kc, vc=vc)
    elif mode == GV_RESID_LN:
        xres = inp["xres"][:R].copy()
        xn = sentinel((R, N), np.float16)
        kw.update(xres=xres, xn=xn, ln_g=inp["ln_g"], ln_b=inp["ln_b"])
        res.update(xres=xres, xn=xn)
        out = None
    elif mode == GV_F32:
        out = sentinel(R * N + GUARD, np.float32)
        kw.update(out=out, ldo=N)
    else:
        out = sentinel(R * N + GUARD, np.float16)
        kw.update(out=out)
    res["out"] = out
    res["path"] = engine.debug_gemv_desc(np.ascontiguousarray(inp["x"][:R]), inp["w"], **kw)
    return res


def check_gv(inp, R, res, name):
    """Checks one R-row result; returns the worst error / bound scale."""
    mode, N = inp["mode"], inp["N"]
    if mode == GV_QKV:
        d = N // 3
        y, rows = inp["y"][:R], inp["rows"][:R]
        assert untouched(res["out"][R * d:]).all(), "guard after q was written"
        s, p = rows[:, 1], rows[:, 2]
        for cache in (res["kc"], res["vc"]):
            hit = np.zeros(cache.shape[:3], bool)
            hit[0, p, s] = True
            assert untouched(cache[~hit]).all(), "a cache entry no row addresses was written"
        return max(check(name + " q", res["out"][:R * d].reshape(R, d), y[:, :d], TOL_GV, quiet=True),
                   check(name + " k", res["kc"][0, p, s], y[:, d:2 * d], TOL_GV, quiet=True),
                   check(name + " v", res["vc"][0, p, s], y[:, 2 * d:], TOL_GV, quiet=True))
    if mode == GV_RESID_LN:
        return max(check(name + " residual", res["xres"], inp["y"][:R], TOL_GV, quiet=True),
                   check(name + " layernorm", res["xn"], inp["xn"][:R], TOL_GV, quiet=True))
    assert untouched(res["out"][R * N:]).all(), "guard after the output was written"
    return check(name, res["out"][:R * N].reshape(R, N), inp["y"][:R], TOL_GV, quiet=True)


GV_CASES = [(m, d) for d in (192, 1280) for m in GV_NAMES] + [("logits", 1280)]


@pytest.mark.parametrize("route", [1, 0], ids=["decoder_route", "skinny"])
@pytest.mark.parametrize("mode,d", GV_CASES, ids=[f"{GV_NAMES.get(m, m)}-d{d}" for m, d in GV_CASES])
def test_decode_gemm_every_row_count(mode, d, route):
    """R = 1..80 through the route the decoder takes (skinny mma.sync kernel up to 16 rows, wgmma with narrow tiles from 17) and
    through the skinny kernel alone (its 7->8 and 9->10 row-group buckets)."""
    inp = gv_inputs(mode, d)
    worst = 0.0
    for R in range(1, 81):
        res = run_gv(inp, R, route)
        assert res["path"] == (1 if route == 1 and R >= 17 else 0), (R, res["path"])
        worst = max(worst, check_gv(inp, R, res, f"gemv {GV_NAMES.get(mode, mode)} d={d} route={route} R={R}"))
    print(f"[measured] gemv {GV_NAMES.get(mode, mode)} d={d} route={route}: max error / bound scale {worst:.3g} (bound {TOL_GV:g})")


# ---- encoder: a chunk's output does not depend on the chunks encoded with it -------------------------------------------------
def encode_each(e, feats):
    return np.stack([e.encode(feats[i:i + 1]).numpy()[0] for i in range(len(feats))])


def assert_batch_invariant(e, n_mels, batches, seed):
    rng = np.random.default_rng(seed)
    feats = (rng.standard_normal((max(batches), n_mels, 3000)) * 0.5).astype(np.float32)
    alone = encode_each(e, feats)
    for B in batches:  # more than 16 chunks: several encoder passes; the flat GEMMs' 128-row tiles straddle chunk boundaries
        together = e.encode(feats[:B]).numpy()
        for i in range(B):
            assert np.array_equal(together[i], alone[i]), f"chunk {i} of {B} differs from the chunk encoded alone"
    from faster_whisper_b200.synthetic import synthetic_audio

    n = 17
    audio = [synthetic_audio(seed + i, s) for i, s in enumerate(np.linspace(0.5, 30.0, n))]
    together = e.encode_audio(audio).numpy()
    for i in range(n):
        alone = e.encode_audio([audio[i]]).numpy()[0]
        assert np.array_equal(together[i], alone), f"encode_audio chunk {i} ({len(audio[i]) / 16000:.1f} s) differs"


def test_encoder_batch_invariance_micro(micro_ml):
    e = engine.Whisper(dims=micro_ml["dims"], weights=micro_ml["weights"], tokens=micro_ml["tokens"], device="cuda")
    assert_batch_invariant(e, micro_ml["dims"].n_mels, (2, 17, 33), seed=5)


def test_encoder_batch_invariance_large_v3():
    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import make_weights

    dims = MODEL_DIMS["large-v3"]
    e = engine.Whisper(dims=dims, weights=make_weights(dims, seed=0), tokens=special_tokens(dims.n_vocab), device="cuda")
    assert_batch_invariant(e, dims.n_mels, (17,), seed=7)


# ---- flash attention: a late maximum ----------------------------------------------------------------------------------------
def test_attention_late_max_in_partial_key_tile():
    """Scores with standard deviation ~8 and every row's largest key in the last, partial 128-key tile (keys 1408..1499): the
    running maximum jumps in the last tile and the earlier tiles' sums are rescaled by about exp(-30)."""
    rng = np.random.default_rng(11)
    B, T, H = 3, 1500, 20
    s = math.sqrt(8.0)
    q = rng.standard_normal((B, T, H, 64)) * s
    k = rng.standard_normal((B, T, H, 64)) * s
    v = rng.standard_normal((B, T, H, 64))
    u = rng.standard_normal((B, H, 64))
    u /= np.linalg.norm(u, axis=-1, keepdims=True)
    q -= np.einsum("bthe,bhe->bth", q, u)[..., None] * u[:, None]  # q orthogonal to u, then a fixed component along it
    q += 4.0 * u[:, None]
    star = rng.integers(1408, T, (B, H))
    for b in range(B):
        for h in range(H):
            k[b, star[b, h], h] = 120.0 * u[b, h]  # score 4 * 120 / 8 = 60 for every query, 7 standard deviations up
    qkv = np.concatenate([q, k, v], 2).reshape(B, T, 3 * H * 64).astype(np.float32)
    got = engine.debug_attention(qkv, H).reshape(B, T, H, 64)
    worst = 0.0
    x = qkv.astype(np.float16).astype(np.float64).reshape(B, T, 3, H, 64)
    for b in range(B):
        for h in range(H):
            sc = x[b, :, 0, h] @ x[b, :, 1, h].T / 8.0
            assert (sc.argmax(1) == star[b, h]).all()
            p = np.exp(sc - sc.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            want = p @ x[b, :, 2, h]
            err = np.abs(got[b, :, h] - want).max()
            assert err < TOL_ATTN, (b, h, err)
            worst = max(worst, err)
    print(f"[measured] attention late max: max |err| {worst:.3g} (bound {TOL_ATTN:g})")
