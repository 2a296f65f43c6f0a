"""A/B of decode-step settings in ONE process: large-v3 (synthetic), B chunks x beam 5, prompt 4 + N new tokens.

For each entry of --configs (environment assignments, e.g. "B2W_STEP=layers") one engine is built with those assignments in force, since
the engine reads its settings when it is created, then one warm-up and `--repeat` timed generate calls; prints the decode time per step
from the engine's stage timers (CUDA events on its stream) and checks that every setting produces the same tokens as the first one.  B2W_LIBRARY=<other build of the C ABI> compares kernel versions on the
same box; with --prof the per-phase device timers of the last step are printed too.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="large-v3")
ap.add_argument("--batch", type=int, default=16)
ap.add_argument("--new-tokens", type=int, default=128)
ap.add_argument("--beam", type=int, default=5)
ap.add_argument("--repeat", type=int, default=2)
ap.add_argument("--configs", default="none", help="';'-separated settings, each a ','-separated list of NAME=VALUE environment assignments ('none' = no assignment)")
ap.add_argument("--compute-type", default="float16")
ap.add_argument("--prof", action="store_true")
a = ap.parse_args()
if a.prof:
    os.environ["B2W_DSTEP_PROF"] = "1"

from faster_whisper_b200 import engine  # noqa: E402
from faster_whisper_b200.config import MODEL_DIMS, special_tokens  # noqa: E402
from faster_whisper_b200.synthetic import make_weights, synthetic_audio  # noqa: E402

dims = MODEL_DIMS[a.model]
st = special_tokens(dims.n_vocab)
weights = make_weights(dims, seed=0)
chunks = [synthetic_audio(i, 30.0) for i in range(a.batch)]
prompt = [st.sot, st.lang_begin, st.transcribe, st.no_timestamps] if dims.is_multilingual else [st.sot, st.no_timestamps]
sup = sorted({st.eot, st.sot, st.transcribe, st.translate, st.sot_prev, st.sot_lm, st.no_speech})
first = None
eng = enc = None
for waves in [w for w in a.configs.split(";") if w]:
    assigned = [kv.split("=", 1) for kv in waves.split(",") if "=" in kv]
    for k, v in assigned:
        os.environ[k] = v
    del eng, enc  # one large-v3 engine at a time
    eng = engine.Whisper(dims=dims, weights=weights, tokens=st, device="cuda", compute_type=a.compute_type)
    for k, _ in assigned:
        os.environ.pop(k, None)
    eng.timing(enable=True)
    enc = eng.encode_audio(chunks)
    eng.sync()
    best = None
    for it in range(1 + a.repeat):
        eng.timing(reset=True)
        res = eng.generate(enc, [prompt] * a.batch, beam_size=a.beam, max_length=len(prompt) + a.new_tokens, suppress_tokens=sup, return_scores=True)
        eng.sync()
        t = eng.timing()
        if it > 0:
            ms = t["decode_ms"] / max(1, t["decode_steps"])
            best = ms if best is None else min(best, ms)
    toks = [r.sequences_ids[0] for r in res]
    if first is None:
        first = toks
    same = sum(x == y for x, y in zip(first, toks))
    print("%s[%s] decode %.4f ms/step (%d steps), tokens identical to the first setting in %d of %d chunks" % (os.environ.get("B2W_LIBRARY", "") and "[other build] ", waves, best, t["decode_steps"], same, len(toks)), flush=True)
