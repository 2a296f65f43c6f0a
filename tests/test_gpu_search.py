"""The on-device search (csrc/search.cu: search_rows + search_update) one step at a time, through ``engine.debug_search``, against a
float64 NumPy reference of the same step written here.

search_rows is checked against float64 arithmetic: the logits processors in CTranslate2's order, the log-softmax and a stable top-2K
(ties to the lower flat index row * V + token).  Tokens must be exact wherever the reference's gap between adjacent ranks exceeds the
score tolerance; inside a smaller gap either order is accepted, but the token sets on both sides of the gap must match.  Tokens whose
keys tie exactly (equal inputs) are not a tolerance case: they must come lowest id first.  Scores (logp + cum) must be within
SCORE_TOL, plus the float32 rounding of the row's largest magnitude for rows far from zero.

search_update is checked exactly: the reference replays CTranslate2's beam step (merge of the rows' candidate lists, finished
hypotheses replaced by secondary candidates, patience, early exit) and the greedy row step on the candidates the device produced, and
every output (history, ancestry, cumulative scores, finished slots, done flags) must be bit-identical.
"""
import numpy as np
import pytest

from conftest import fake_logits_numpy
from faster_whisper_b200 import engine
from faster_whisper_b200.config import special_tokens
from faster_whisper_b200.synthetic import custom_dims
from oracle.whisper_oracle import WhisperOracle

LOWEST = float(np.finfo(np.float32).min)
F32_EPS = 2.0**-23
SCORE_TOL = 1e-5       # logp + cum, rows of moderate magnitude (largest error measured on an H100 80GB HBM3 at 700 W: 3.5e-6)
NO_SPEECH_RTOL = 1e-5  # relative, softmax probability of <|nospeech|>
VOCABS = [51864, 51865, 51866]
MAXF = engine.MAX_FINISHED

# largest error measured against each bound, printed at the end of the module (pytest -s)
WORST = {"score": 0.0, "score_large_rows": 0.0, "no_speech_rel": 0.0, "sampling_score": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nsearch step: largest error against each bound:", {k: float(f"{v:.3g}") for k, v in WORST.items()})


def model(V):
    dims = custom_dims(n_vocab=V)
    return dims, special_tokens(V)


# ---- float64 reference -------------------------------------------------------------------------------------------------
def _lse(x):
    m = x.max()
    return m + np.log(np.exp(x - m).sum())


def ref_process(x32, step, h, o, tk, timestamp_rules):
    """Processed logits of one row in float64, CTranslate2's order: repetition penalty, no-repeat n-gram, suppress_tokens,
    suppress_blank, Whisper timestamp rules.  Masked entries hold LOWEST.  Also returns the timestamp-mass rule's margin
    (timestamp log-prob minus best text log-prob; None where the rule is not evaluated)."""
    x = x32.astype(np.float64)
    h = [int(v) for v in h]
    rp = float(np.float32(o.get("repetition_penalty", 1.0)))
    if rp != 1.0 and h:
        ids = np.unique(h)
        v = x32[ids].astype(np.float64)
        x[ids] = np.where(v < 0, v * rp, v / rp)
    ng = o.get("no_repeat_ngram_size", 0)
    if ng > 0 and len(h) >= ng:
        prefix = h[len(h) - ng + 1:]
        for s in range(len(h) - ng + 1):
            if h[s:s + ng - 1] == prefix:
                x[h[s + ng - 1]] = LOWEST
    sup = [int(t) for t in (o.get("suppress_tokens", (-1,)) or []) if int(t) >= 0]
    x[sup] = LOWEST
    if o.get("suppress_blank", True) and step == 0:
        x[[220, tk.eot]] = LOWEST
    margin = None
    if timestamp_rules:
        ts0, eot = tk.timestamp_begin, tk.eot
        x[tk.no_timestamps] = LOWEST
        if step == 0:
            x[:ts0] = LOWEST
            mi = o.get("max_initial_timestamp_index", 50)
            if mi >= 0:
                x[ts0 + mi + 1:] = LOWEST
        else:
            last_ts = h[-1] >= ts0
            penult_ts = len(h) < 2 or h[-2] >= ts0
            if last_ts:
                if penult_ts:
                    x[ts0:] = LOWEST
                else:
                    x[:eot] = LOWEST
            stamps = [t for t in h if t >= ts0]
            if stamps:
                t_last = stamps[-1] if (last_ts and not penult_ts) else stamps[-1] + 1
                x[ts0:t_last] = LOWEST
            live = x > LOWEST / 2
            lse = _lse(x[live])
            ts = x[ts0:][live[ts0:]]
            ts_lp = _lse(ts) - lse if ts.size else -np.inf
            text_lp = x[:ts0].max() - lse
            margin = ts_lp - text_lp
            if ts_lp > text_lp:
                x[:ts0] = LOWEST
    return x, margin


def ref_logp(x):
    live = x > LOWEST / 2
    return x - _lse(x[live])


def gumbel64(seed, row, step, V):
    u = (WhisperOracle.gumbel_bits(seed, row, step, V).astype(np.float64) + 0.5) / 8388608.0
    return -np.log(-np.log(u))


def check_topk(got_tok, got_sc, key, score, tol, what):
    """Device top-n (tokens, scores) of one row against float64 ranking keys and expected scores (see the module docstring)."""
    nc = len(got_tok)
    V = key.shape[0]
    got_tok = np.asarray(got_tok, np.int64)
    assert len(set(got_tok.tolist())) == nc, (what, "duplicate candidates", got_tok)
    assert np.all((got_tok >= 0) & (got_tok < V)), (what, got_tok)
    order = np.lexsort((np.arange(V), -key))
    ks = key[order]
    fin = np.isfinite(ks)
    with np.errstate(invalid="ignore"):
        gaps = np.where(fin[:-1] & fin[1:], ks[:-1] - ks[1:], np.where(fin[:-1] == fin[1:], 0.0, np.inf))
    block = np.concatenate([[0], np.cumsum(gaps > tol)])  # block id of each sorted position
    block_of_tok = np.empty(V, np.int64)
    block_of_tok[order] = block
    bad = np.flatnonzero(block_of_tok[got_tok] != block[:nc])
    assert bad.size == 0, (what, "rank", int(bad[0]), "got", got_tok[: bad[0] + 3].tolist(), "want", order[: bad[0] + 3].tolist(),
                           "keys", ks[: bad[0] + 3].tolist())
    # exact ties: lowest ids first, in id order
    kg = key[got_tok]
    for u in np.unique(kg):
        pos = np.flatnonzero(kg == u)
        if pos.size == 1 and np.count_nonzero(key == u) == 1:
            continue
        group = np.flatnonzero(key == u)
        assert got_tok[pos].tolist() == group[: pos.size].tolist(), (what, "exact tie", got_tok[pos].tolist(), group[: pos.size].tolist())
    # scores
    want = score[got_tok]
    masked = want <= -1e38
    assert np.all(np.isfinite(got_sc[masked])) and np.all(got_sc[masked] <= -1e38), (what, "masked candidates", got_sc[masked])
    err = np.abs(got_sc[~masked].astype(np.float64) - want[~masked])
    e = float(err.max()) if err.size else 0.0
    assert e <= tol, (what, "score error", e, tol)
    return e


def ref_rows(lg, prompt, t, hist, cum, o, tk):
    """Per-row float64 keys / expected scores of search_rows, and the timestamp margins."""
    n, K, V = lg.shape
    beam = o.get("beam_size", 5) > 1
    sampling = not beam and o.get("sampling_topk", 1) == 0
    T = float(np.float32(o.get("sampling_temperature", 1.0)))
    ts_rules = tk.no_timestamps not in list(prompt)
    rows = []
    for b in range(n):
        for k in range(K):
            x, margin = ref_process(lg[b, k], t, hist[b, k], o, tk, ts_rules)
            lp = ref_logp(x)
            masked = x <= LOWEST / 2
            if beam:
                key = lp + float(cum[b, k])
                score = key
            elif sampling:
                score = lp / T
                key = np.where(masked, -np.inf, score + gumbel64(o.get("seed", 0), b * K + k, t, V))
            else:
                key = score = lp
            score = np.where(masked, LOWEST, score)
            rows.append((key, score, margin, float(np.abs(lg[b, k][~masked]).max(initial=0.0)) + abs(float(cum[b, k]))))
    return rows


def ref_update(out, prompt, t, st_in, o, tk, V):
    """CTranslate2's beam step / the greedy row step on the device's candidates; returns the expected state after the step."""
    n, K = st_in["cum"].shape
    P = len(prompt)
    pos = P - 1 + t
    beam = o.get("beam_size", 5) > 1
    max_steps = min(o.get("max_length", 448), 448) - P
    is_last = t + 1 >= max_steps
    eot = tk.eot
    cs, ct = out["cand_score"], out["cand_tok"]
    exp = {k: np.array(v, copy=True) for k, v in st_in.items()}
    exp["fin_tok"] = np.full((n, MAXF, t + 1), -1, np.int32)
    new_hist = np.zeros((n, K, t + 1), np.int32)
    new_anc = np.zeros((n, K, pos + 1), np.uint8)
    new_cum = np.zeros((n, K), np.float32)
    tokens_in = np.zeros((n, K), np.int32)
    n_done = st_in["n_done"]
    if beam:
        patience, lp = o.get("patience", 1.0), o.get("length_penalty", 1.0)
        max_finished = max(1, int(np.floor(K * patience + 0.5)))
        early = patience == 1 and lp == 0
        num_hyp = o.get("num_hypotheses", 1)
        ncand = 2 * K
    for b in range(n):
        chunk_done = st_in["done"][b] != 0
        fins = []
        if beam:
            nrows = 1 if t == 0 else K
            head = [0] * nrows
            c_score, c_tok, c_beam = [], [], []
            for _ in range(ncand):
                bi, bs, bflat = -1, 0.0, 0
                for i in range(nrows):
                    if head[i] >= ncand:
                        continue
                    sc = cs[b, i, head[i]]
                    flat = i * V + int(ct[b, i, head[i]])
                    if bi < 0 or sc > bs or (sc == bs and flat < bflat):
                        bi, bs, bflat = i, sc, flat
                c_score.append(bs)
                c_beam.append(bi)
                c_tok.append(int(ct[b, bi, head[bi]]))
                head[bi] += 1
            secondary, top_finished = K, False
            nfin = int(st_in["fin_count"][b])
            parent, newtok, newcum = [], [], []
            for k in range(K):
                nx = k
                tok = c_tok[k]
                if (tok == eot or is_last) and not chunk_done:
                    if k == 0:
                        top_finished = True
                    assert nfin < MAXF
                    fins.append((c_beam[k], nfin, tok if tok != eot else -1, c_score[k]))
                    nfin += 1
                    for j in range(secondary, ncand):
                        if c_tok[j] != eot:
                            nx, secondary = j, j + 1
                            break
                parent.append(c_beam[nx])
                newtok.append(c_tok[nx])
                newcum.append(c_score[nx])
            if not chunk_done:
                exp["fin_count"][b] = nfin
                if is_last:
                    fin = True
                elif early:
                    fin = top_finished and nfin >= num_hyp
                else:
                    fin = nfin >= max_finished
                if fin:
                    exp["done"][b] = 1
                    n_done += 1
        else:
            parent, newtok, newcum = list(range(K)), [], []
            ndone_rows = 0
            for k in range(K):
                tok, sc = int(ct[b, k, 0]), np.float32(cs[b, k, 0])
                newtok.append(tok)
                cumv = np.float32(st_in["cum"][b, k])
                if st_in["fin_len"][b, k] < 0:
                    cumv = np.float32(cumv + sc)
                    if tok == eot or is_last:
                        fins.append((k, k, tok if tok != eot else -1, cumv))
                        ndone_rows += 1
                else:
                    ndone_rows += 1
                newcum.append(cumv)
            if not chunk_done and ndone_rows == K:
                exp["fin_count"][b] = K
                exp["done"][b] = 1
                n_done += 1
        for src, slot, extra, sc in fins:
            seq = list(st_in["hist"][b, src, :t]) + ([extra] if extra >= 0 else [])
            exp["fin_tok"][b, slot, : len(seq)] = seq
            exp["fin_len"][b, slot] = len(seq)
            exp["fin_score"][b, slot] = sc
        for k in range(K):
            pk = parent[k]
            new_hist[b, k, :t] = st_in["hist"][b, pk, :t]
            new_hist[b, k, t] = newtok[k]
            new_anc[b, k, :pos] = st_in["anc"][b, pk, :pos]
            new_anc[b, k, pos] = pk
            new_cum[b, k] = newcum[k]
            tokens_in[b, k] = newtok[k]
    exp.update(hist=new_hist, anc=new_anc, cum=new_cum, tokens_in=tokens_in, pos=np.full((n, K), pos + 1, np.int32), n_done=n_done)
    return exp


def run_step(V, logits, prompt, t, *, hist=None, anc=None, cum=None, done=None, fin_count=None, fin_len=None, fin_score=None,
             n_done=0, **o):
    """One device step checked against the reference; returns (device outputs, per-row reference tuples)."""
    dims, tk = model(V)
    logits = np.ascontiguousarray(logits, np.float32)
    n, K, _ = logits.shape
    P = len(prompt)
    rng = np.random.default_rng(t + 17 * K)
    st_in = dict(
        hist=np.zeros((n, K, t), np.int32) if hist is None else np.asarray(hist, np.int32).reshape(n, K, t),
        anc=rng.integers(0, K, (n, K, P - 1 + t)).astype(np.uint8) if anc is None else np.asarray(anc, np.uint8),
        cum=np.zeros((n, K), np.float32) if cum is None else np.asarray(cum, np.float32).reshape(n, K),
        done=np.zeros(n, np.int32) if done is None else np.asarray(done, np.int32),
        fin_count=np.zeros(n, np.int32) if fin_count is None else np.asarray(fin_count, np.int32),
        fin_len=np.full((n, MAXF), -1, np.int32) if fin_len is None else np.asarray(fin_len, np.int32),
        fin_score=np.zeros((n, MAXF), np.float32) if fin_score is None else np.asarray(fin_score, np.float32),
        n_done=n_done)
    out = engine.debug_search(dims, tk, logits, prompt, t, **{k: v for k, v in st_in.items()}, **o)
    rows = ref_rows(logits, prompt, t, st_in["hist"], st_in["cum"], o, tk)
    beam = o.get("beam_size", 5) > 1
    sampling = not beam and o.get("sampling_topk", 1) == 0
    for r, (key, score, _, mag) in enumerate(rows):
        b, k = divmod(r, K)
        tol = SCORE_TOL + 2 * F32_EPS * mag
        if sampling:  # the log-prob's error scaled by 1 / temperature
            tol *= max(1.0, 1.0 / o.get("sampling_temperature", 1.0))
        e = check_topk(out["cand_tok"][b, k], out["cand_score"][b, k], key, score, tol, (b, k))
        name = "sampling_score" if sampling else ("score_large_rows" if mag > 100 else "score")
        WORST[name] = max(WORST[name], e)
    exp = ref_update(out, prompt, t, st_in, o, tk, V)
    for name in ("hist", "anc", "cum", "tokens_in", "pos", "done", "n_done", "fin_count", "fin_len", "fin_score", "fin_tok"):
        np.testing.assert_array_equal(np.asarray(out[name]), np.asarray(exp[name]), err_msg=name)
    return out, rows


def base_logits(rng, n, K, V, lo=-4.0, hi=4.0):
    return rng.uniform(lo, hi, (n, K, V)).astype(np.float32)


# ---- CPU: the reference against the oracle's processors -----------------------------------------------------------------
def test_reference_matches_oracle_processors(micro):
    o_ = micro["oracle"]
    tk = micro["tokens"]
    V = micro["dims"].n_vocab
    ts0 = tk.timestamp_begin
    rng = np.random.default_rng(3)
    for case in range(24):
        step = int(rng.integers(0, 6))
        ts = bool(case % 2)
        h = [int(v) for v in rng.choice([5, 6, 7, 300, ts0 + 3, ts0 + 9, V - 1], step)]
        o = dict(repetition_penalty=[1.0, 1.3, 0.7][case % 3], no_repeat_ngram_size=case % 4,
                 suppress_tokens=[0, 11, V - 2], suppress_blank=bool(case % 5), max_initial_timestamp_index=[-1, 0, 50][case % 3])
        x32 = rng.normal(0, 3, V).astype(np.float32)
        x32[ts0:] += np.float32(rng.uniform(-8, 2))
        mine, _ = ref_process(x32, step, h, o, tk, ts)
        want = x32[None].copy()
        od = dict(repetition_penalty=o["repetition_penalty"], no_repeat_ngram_size=o["no_repeat_ngram_size"],
                  suppress_ids=np.asarray(sorted(o["suppress_tokens"]), np.int64), suppress_blank=o["suppress_blank"],
                  timestamp_rules=ts, max_initial_timestamp_index=o["max_initial_timestamp_index"])
        o_._process_logits(want, step, [h], od)
        assert np.array_equal(mine <= LOWEST / 2, want[0] <= LOWEST / 2), case
        live = mine > LOWEST / 2
        np.testing.assert_allclose(ref_logp(mine)[live], o_._log_softmax(want)[0][live], atol=2e-5, err_msg=str(case))
    # the float64 Gumbel keys are the oracle's noise
    np.testing.assert_allclose(gumbel64(1234, 3, 2, V), WhisperOracle.gumbel_noise(1234, 3, 2, V), rtol=1e-6, atol=1e-6)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_static_masks(V):
    dims, tk = model(V)
    rng = np.random.default_rng(V)
    lg = base_logits(rng, 2, 2, V)
    lg[..., 0] = 9.0
    lg[..., V - 1] = 8.5
    lg[..., 220] = 8.0
    lg[..., tk.eot] = 7.5
    prompt = [tk.sot, tk.no_timestamps]
    for t in (0, 1):
        out, _ = run_step(V, lg, prompt, t, hist=np.full((2, 2, t), 300), beam_size=2, max_length=30, suppress_tokens=[-1, 0, V - 1, 17])
        toks = out["cand_tok"].reshape(-1)
        assert 0 not in toks and V - 1 not in toks
        assert (220 in toks) == (t == 1) and (tk.eot in toks) == (t == 1)


@gpu
@pytest.mark.parametrize("rp", [1.3, 0.7])
@pytest.mark.parametrize("V", VOCABS)
def test_repetition_penalty(V, rp):
    dims, tk = model(V)
    rng = np.random.default_rng(int(rp * 10) + V)
    K, n = 8, 2
    prompt = [tk.sot, tk.no_timestamps]
    for t in (3, 64, 445):
        lg = base_logits(rng, n, K, V, -12, -10)
        hist = rng.integers(1000, 2000, (n, K, t))
        # repeated many times, positive / negative / zero logits, and a suppressed token in the history
        special = [2500, 2501, 2502, 2503, 2504]
        for i, v in enumerate(special):
            hist[:, :, i % t] = v
        hist[:, :, t // 2:] = 2500
        lg[..., 2500] = 3.0
        lg[..., 2501] = -0.5
        lg[..., 2502] = 0.0
        lg[..., 2503] = 2.0
        lg[..., 2504] = 9.0  # suppressed: stays masked whatever the penalty
        lg[..., 3000:3010] = np.linspace(3.5, -1.0, 10)  # unpenalised competitors between the penalised values
        run_step(V, lg, prompt, t, hist=hist, cum=rng.uniform(-20, 0, (n, K)), beam_size=K, max_length=448, repetition_penalty=rp,
                 suppress_tokens=[2504])


@gpu
@pytest.mark.parametrize("ng", [1, 2, 3])
@pytest.mark.parametrize("V", VOCABS)
def test_no_repeat_ngram(V, ng):
    dims, tk = model(V)
    rng = np.random.default_rng(ng + V)
    a, b, c, d, e = 400, 401, 402, 403, 404
    t = 8
    hists = [
        [a, b, c, a, b, d, a, b],  # the prefix (a, b) matches at two places
        [a, a, a, a, a, a, a, a],  # overlapping n-grams
        [e, e, e, e, e, a, b, c],
        [c, d, e, a, b, c, d, e],
        [a, b, a, b, a, b, a, b],
    ]
    K = len(hists)
    lg = base_logits(rng, 1, K, V, -6, -4)
    lg[..., [a, b, c, d, e]] = [5.0, 4.5, 4.0, 3.5, 3.0]
    prompt = [tk.sot, tk.no_timestamps]
    run_step(V, lg, prompt, t, hist=np.asarray(hists)[None], beam_size=1, num_hypotheses=K, no_repeat_ngram_size=ng, max_length=40)
    # fewer generated tokens than n, and exactly n
    for tt in (ng - 1, ng):
        run_step(V, lg[:, :2], prompt, tt, hist=np.full((1, 2, tt), a), beam_size=2, no_repeat_ngram_size=ng, max_length=40)


@gpu
@pytest.mark.parametrize("mi", [-1, 0, 50])
@pytest.mark.parametrize("V", VOCABS)
def test_timestamp_rules_first_step(V, mi):
    dims, tk = model(V)
    ts0 = tk.timestamp_begin
    rng = np.random.default_rng(V + mi)
    lg = base_logits(rng, 1, 2, V, -2, 2)
    lg[..., ts0:] = np.linspace(0, 6, V - ts0, dtype=np.float32)  # later stamps preferred: the upper cut decides the winner
    lg[..., 100] = 12.0
    out, _ = run_step(V, lg, [tk.sot], 0, beam_size=2, max_length=30, max_initial_timestamp_index=mi, return_no_speech_prob=True)
    top = int(out["cand_tok"][0, 0, 0])
    assert top == (V - 1 if mi < 0 else ts0 + mi)


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_timestamp_rules(V):
    dims, tk = model(V)
    ts0, eot = tk.timestamp_begin, tk.eot
    nts = V - ts0
    rng = np.random.default_rng(V)
    t = 4
    hists = [
        [ts0 + 2, 100, ts0 + 5, ts0 + 6],  # last two are stamps: text only
        [ts0 + 1, 100, 200, ts0 + 7],      # a lone stamp: a stamp >= it, or EOT
        [ts0 + 3, 100, 200, 300],          # last is text: stamps after the last one
        [100, V - 1, 200, 300],            # last stamp V-1: every stamp masked, no timestamp mass
        [100, 200, 300, 400],              # timestamp mass beats the best text token (margin +0.5)
        [100, 200, 300, 401],              # ... and does not (margin -0.5)
    ]
    K = len(hists)
    lg = base_logits(rng, 1, K, V, -9, -7)
    lg[0, :, 500] = 5.0
    lg[0, :, eot] = 1.0
    lg[0, :, ts0 + 7] = 4.0
    lg[0, :, ts0:ts0 + 7] = 6.0
    for k, margin in ((4, 0.5), (5, -0.5)):
        # exp(ts) * nts = exp(5 + margin) against the text token at 5 (every other entry is negligible)
        lg[0, k, ts0:] = 5.0 + margin - np.log(nts)
    out, rows = run_step(V, lg, [tk.sot], t, hist=np.asarray(hists)[None], beam_size=1, num_hypotheses=K, max_length=40)
    for k, (_, _, m, _) in enumerate(rows):
        assert m is not None and (m == -np.inf or abs(m) >= 1e-3), (k, m)
    assert rows[3][2] == -np.inf
    assert rows[4][2] > 1e-3 and rows[5][2] < -1e-3
    got = out["cand_tok"][0, :, 0].tolist()
    assert got[0] == 500 and got[1] == ts0 + 7 and got[3] == 500 and got[4] >= ts0 and got[5] == 500, got
    # one generated token, a stamp: "penultimate" counts as a stamp, so the next token is text
    out, _ = run_step(V, lg[:, :2], [tk.sot], 1, hist=np.full((1, 2, 1), ts0 + 3), beam_size=1, num_hypotheses=2, max_length=40)
    assert out["cand_tok"][0, 0, 0] == 500


def topk_rows(rng, K, V, n_rows):
    """Rows that stress the row top-2K extraction, cycled over the rows."""
    nc = 2 * K if K > 1 else 1
    rows = []
    for i in range(n_rows):
        x = rng.uniform(-4, 4, V).astype(np.float32)
        kind = i % 8
        if kind == 0:  # plateau of 40 equal maxima
            x[rng.choice(V, 40, replace=False)] = 7.0
        elif kind == 1:  # whole row constant
            x[:] = 0.25
        elif kind == 2:  # the top 2K in one thread's strided slice (ids congruent mod 1024): its second, then its rescan
            ids = (rng.integers(0, 1024) + 1024 * np.arange(nc + 3)) % V
            x[ids] = 10.0 - 0.125 * np.arange(ids.size)
        elif kind == 3:  # the top 2K inside one warp's slice
            w = int(rng.integers(0, 32))
            ids = rng.choice(np.flatnonzero((np.arange(V) % 1024) // 32 == w), nc + 3, replace=False)
            x[ids] = 10.0 - 0.0625 * np.arange(ids.size)
        elif kind == 4:  # the winner at V-1
            x[V - 1] = 9.0
            x[V - 2] = 8.0
        elif kind == 5:  # large magnitudes
            x = (1e4 + rng.uniform(-20, 20, V)).astype(np.float32)
        elif kind == 6:
            x = (-1e4 + rng.uniform(-20, 20, V)).astype(np.float32)
        else:  # one token 60 above the rest
            x[int(rng.integers(0, V))] = x.max() + 60.0
        rows.append(x)
    return np.stack(rows)


@gpu
@pytest.mark.parametrize("K", [1, 2, 5, 16])
@pytest.mark.parametrize("V", VOCABS)
def test_topk_extraction(V, K):
    dims, tk = model(V)
    rng = np.random.default_rng(V * 7 + K)
    prompt = [tk.sot, tk.no_timestamps]
    opts = dict(beam_size=K, max_length=60) if K > 1 else dict(beam_size=1, max_length=60)
    n = max(2, -(-8 // K) + 1)
    lg = topk_rows(rng, K, V, n * K).reshape(n, K, V)
    cum = rng.uniform(-3, 0, (n, K)).astype(np.float32)
    # the last chunk: every row the same logits and the same cumulative score, so candidates tie across beams
    lg[-1] = lg[-1, 0]
    cum[-1] = cum[-1, 0]
    run_step(V, lg, prompt, 1, hist=rng.integers(0, 50000, (n, K, 1)), cum=cum, **opts)
    run_step(V, lg, prompt, 0, **opts)
    # exactly 2K-1 live tokens (one for greedy), the rest suppressed: the last candidate is a masked one
    live = np.sort(rng.choice(V, 2 * K - 1, replace=False))
    sup = np.setdiff1d(np.arange(V), live)
    out, _ = run_step(V, lg[:1], prompt, 1, hist=np.full((1, K, 1), 7), cum=cum[:1], suppress_tokens=sup.tolist(), **opts)
    if K > 1:
        assert np.all(out["cand_score"][0, :, -1] <= -1e38) and np.all(np.isfinite(out["cand_score"]))
        assert np.all(out["cand_tok"][0, :, -1] == sup[0])


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_no_speech_probability(V):
    dims, tk = model(V)
    rng = np.random.default_rng(V + 5)
    lg = base_logits(rng, 3, 2, V, -6, 6)
    lg[0, :, tk.no_speech] = 8.0
    lg[1, :, tk.no_speech] = -3.0
    lg[2, :, 77] = 30.0
    for prompt in ([tk.sot], [tk.sot_prev, 11, 12, tk.sot]):
        out, _ = run_step(V, lg, prompt, 0, beam_size=2, max_length=30, return_no_speech_prob=True, suppress_tokens=[tk.no_speech])
        want = np.array([WhisperOracle._softmax64(lg[b, 0][None])[0, tk.no_speech] for b in range(3)])
        rel = np.abs(out["no_speech"] - want) / want
        WORST["no_speech_rel"] = max(WORST["no_speech_rel"], float(rel.max()))
        assert rel.max() < NO_SPEECH_RTOL, (rel, out["no_speech"], want)
    # the probability comes from the step whose fed token is <|startoftranscript|>
    out, _ = run_step(V, lg, [tk.sot, tk.no_timestamps], 0, beam_size=2, max_length=30, return_no_speech_prob=True)
    assert np.all(out["no_speech"] == 0)


@gpu
@pytest.mark.parametrize("T", [0.6, 1.5])
@pytest.mark.parametrize("V", VOCABS)
def test_sampling(V, T):
    dims, tk = model(V)
    rng = np.random.default_rng(V + int(T * 10))
    K = 5
    lg = base_logits(rng, 2, K, V, -3, 3)
    lg[0, :, 500:503] = 6.0
    for t in (0, 3):
        run_step(V, lg, [tk.sot, tk.no_timestamps], t, hist=rng.integers(0, 50000, (2, K, t)), cum=rng.uniform(-5, 0, (2, K)),
                 beam_size=1, num_hypotheses=K, sampling_topk=0, sampling_temperature=T, seed=99, max_length=30,
                 suppress_tokens=[500])


# ---- search_update transitions --------------------------------------------------------------------------------------------
def eot_logits(rng, n, K, V, eot, ranks):
    """Logits whose row k has EOT at rank ranks[b][k] (None: EOT low)."""
    lg = base_logits(rng, n, K, V, -8, -6)
    for b in range(n):
        for k in range(K):
            top = rng.choice(np.arange(1000, 5000), 2 * K + 2, replace=False)
            lg[b, k, top] = np.linspace(4.0, 2.0, top.size)
            r = ranks[b][k]
            if r is not None:
                lg[b, k, eot] = np.float32(4.0 - (2.0 / (top.size - 1)) * r + 0.01)
    return lg


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_update_eot_positions_and_done_chunks(V):
    dims, tk = model(V)
    rng = np.random.default_rng(V + 11)
    K, n, t = 4, 4, 5
    # chunk 0: EOT is the best candidate; chunk 1: EOT in the middle of the top K; chunk 2: EOT high in every row (several of the
    # top K finish); chunk 3: already done, next to live ones (writes nothing to its finished list)
    ranks = [[0, None, None, None], [None, 2, None, 1], [0, 0, 1, 0], [0, 0, 0, 0]]
    lg = eot_logits(rng, n, K, V, tk.eot, ranks)
    cum = np.repeat(rng.uniform(-4, -3, (n, 1)), K, 1) + rng.uniform(-0.05, 0, (n, K))
    cum[0, 0] += 0.5  # chunk 0's best candidate is row 0's EOT
    fin_len = np.full((n, MAXF), -1)
    fin_len[3, :3] = [2, 3, 4]
    common = dict(hist=rng.integers(0, 50000, (n, K, t)), cum=cum, done=[0, 0, 0, 1], fin_count=[2, 0, 5, 3], fin_len=fin_len,
                  fin_score=rng.uniform(-9, -1, (n, MAXF)), n_done=1, beam_size=K, max_length=60)
    for extra in (dict(), dict(patience=1.0, length_penalty=0.0), dict(patience=1.5, num_hypotheses=2), dict(max_length=3 + t)):
        out, _ = run_step(V, lg, [tk.sot, tk.no_timestamps], t, **{**common, **extra})
        assert out["fin_count"][3] == 3 and out["fin_len"][3, :4].tolist() == [2, 3, 4, -1]
    # patience 1, length penalty 0: the chunk whose best candidate is EOT stops once num_hypotheses are finished
    out, _ = run_step(V, lg, [tk.sot, tk.no_timestamps], t, **{**common, "patience": 1.0, "length_penalty": 0.0})
    assert out["done"][0] == 1 and out["done"][1] == 0


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_update_keeps_every_finished_hypothesis(V):
    """K = 16, patience 2 (stop at 32 finished), 31 finished already, EOT the best token of every row: 16 more finish in this step
    and all 47 are kept."""
    dims, tk = model(V)
    rng = np.random.default_rng(V + 13)
    K, t = 16, 9
    lg = eot_logits(rng, 1, K, V, tk.eot, [[0] * K])
    cum = np.full((1, K), -5.0, np.float32) + rng.uniform(-0.005, 0, (1, K)).astype(np.float32)
    fin_len = np.full((1, MAXF), -1)
    fin_len[0, :31] = rng.integers(1, t + 1, 31)
    out, _ = run_step(V, lg, [tk.sot, tk.no_timestamps], t, hist=rng.integers(0, 50000, (1, K, t)), cum=cum, fin_count=[31],
                      fin_len=fin_len, fin_score=rng.uniform(-9, -1, (1, MAXF)), beam_size=K, patience=2.0, num_hypotheses=16,
                      max_length=60)
    assert out["fin_count"][0] == 47 and out["done"][0] == 1 and out["n_done"] == 1
    assert np.all(out["fin_len"][0, 31:47] == t) and out["fin_len"][0, 47] == -1


@gpu
@pytest.mark.parametrize("V", VOCABS)
def test_update_greedy_rows_finish_at_different_steps(V):
    dims, tk = model(V)
    rng = np.random.default_rng(V + 17)
    K, t = 4, 6
    lg = eot_logits(rng, 2, K, V, tk.eot, [[0, None, 0, None], [0, 0, None, 0]])
    fin_len = np.full((2, MAXF), -1)
    fin_len[0, 1] = 3  # row 1 of chunk 0 finished earlier; row 3 goes on
    fin_len[1, 2] = 5  # chunk 1: the last live rows finish now, so the chunk is done
    out, _ = run_step(V, lg, [tk.sot, tk.no_timestamps], t, hist=rng.integers(0, 50000, (2, K, t)), cum=rng.uniform(-5, 0, (2, K)),
                      fin_len=fin_len, fin_score=rng.uniform(-9, -1, (2, MAXF)), beam_size=1, num_hypotheses=K, max_length=40)
    assert out["done"].tolist() == [0, 1] and out["fin_count"][1] == K
    assert out["fin_len"][0, :4].tolist() == [t, 3, t, -1]
    # the last step finishes every row, with its token kept
    out, _ = run_step(V, lg, [tk.sot, tk.no_timestamps], t, hist=rng.integers(0, 50000, (2, K, t)), beam_size=1, num_hypotheses=K,
                      max_length=3 + t)
    assert out["done"].tolist() == [1, 1]


# ---- the finished-hypothesis cap over a whole generate call (fake logits, against the oracle) --------------------------------
def _search_case(eng, m, prompts, **kw):
    st = m["tokens"]
    fl = fake_logits_numpy(m["dims"].n_vocab, st.timestamp_begin, st.eot)
    want = m["oracle"].generate(None, prompts, fake_logits=fl, return_scores=True, return_no_speech_prob=False, **kw)
    got = eng.generate(None, prompts, _fake_logits=True, return_scores=True, **kw)
    for w, g in zip(want, got):
        assert g.sequences_ids == w.sequences_ids, (kw, g.sequences_ids, w.sequences_ids)
        assert np.allclose(g.scores, w.scores, rtol=1e-4, atol=1e-4), (g.scores, w.scores)


@pytest.fixture(scope="module")
def eng(micro):
    return engine.Whisper(dims=micro["dims"], weights=micro["weights"], tokens=micro["tokens"], device="cuda")


@gpu
def test_beam16_patience2_keeps_every_finished_hypothesis(eng, micro):
    """35 and 38 hypotheses finish in these chunks; several of the best 16 finish after the 32nd."""
    st = micro["tokens"]
    for tok in (101, 321):
        _search_case(eng, micro, [[st.sot, st.no_timestamps, tok]], beam_size=16, patience=2.0, num_hypotheses=16, max_length=60,
                     length_penalty=1.0)


@gpu
def test_beam16_with_timestamps(eng, micro):
    st = micro["tokens"]
    _search_case(eng, micro, [[st.sot, 100], [st.sot, 101]], beam_size=16, patience=1.5, num_hypotheses=4, max_length=40)
