#!/usr/bin/env python
"""Benchmark of the hot path BASELINE.json names: log-mel -> encoder -> beam-5 decoder, large-v3 fp16, 30 s chunks.

    python bench.py --gpus N --steps K --warmup W            # our engine (one process per GPU under torchrun for N>1)
    python bench.py --impl reference --gpus N --steps K ...  # the CPU restatement of the reference path (rank 0 only)

A *step* is one pass of the hot path over one batch of synthetic 30 s chunks on every GPU:
``--workload batched`` (default, BASELINE.json configs[2], the configuration configs[4] shards) = 16 chunks through one
generate() call (``--compute-type int8_float16`` = configs[3]); ``--workload single`` (configs[1]) = one chunk, beam_size=5.
The default line also carries the single-chunk measurement of the same process under ``single_chunk``.
Weak scaling: per-GPU work is fixed.
Decode length is pinned (SURVEY.md §8d): prompt of 4 tokens, exactly 128 new tokens (EOT in suppress_tokens).

``--dump-outputs DIR`` writes what the timed engine path returned in its last step (token ids, scores, no-speech
probabilities, a fixed seeded sample of the encoder output) as ``DIR/<name>.npy``; the inputs depend only on the
arguments, so two builds can be compared output for output.

Prints ONE JSON line (rank 0).  ``value`` = audio seconds per second through the engine calls (encode_audio + generate; the
1.92 MB/chunk PCM upload is inside, see ``stages_ms.h2d``), timed with CUDA events on the engine's stream around the K steps
(barrier + sync on both sides, max over ranks; the host wall clock of the same region is in ``host_wall_ms_per_step``);
``e2e`` = the same metric through the public API (``BatchedInferencePipeline.transcribe`` on a host NumPy waveform, segments
consumed); ``roofline`` = decode-step HBM roofline (algorithmic bytes W + B*X + R*t*S per step over the CUDA-event time of the
decode stage on the engine's stream).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "audio-sec/s (RTF) large-v3 fp16 beam=5, 30s chunks"
NEW_TOKENS = 128


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return dict(hbm_gbs=d["hbm_gbs"], tflops=d.get("bf16_tflops_sustained", d["bf16_tflops"]), source="measured")
    # NVIDIA H100 SXM data sheet: 3.35 TB/s HBM3, 989 TFLOP/s dense FP16/BF16 (a 700 W card; a lower power limit lowers the reachable rate)
    return dict(hbm_gbs=3350.0, tflops=989.0, source="H100 SXM data sheet")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index = index
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "200"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except OSError:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, smax, reasons = [], [], set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                smax.append(float(f[1]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def dist_env():
    return int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))


# ----------------------------------------------------------------------------------------------------------------
# CPU baseline: the oracle (a port of the reference path; CTranslate2 itself is not installable here, DESIGN.md)
# ----------------------------------------------------------------------------------------------------------------
def host_threads(cap: int = 16) -> int:
    """Threads the CPU arm uses: the cores this process may actually run on (affinity and cgroup quota), capped — on a
    128-core box an uncapped torch thread pool ran this path 10x slower than 8 threads do."""
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except (AttributeError, OSError):
        pass
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            with open(path) as f:
                parts = f.read().split()
            if path.endswith("cpu.max"):
                if parts[0] != "max":
                    n = min(n, max(1, int(int(parts[0]) / int(parts[1]))))
            else:
                q = int(parts[0])
                if q > 0:
                    with open("/sys/fs/cgroup/cpu/cpu.cfs_period_us") as f2:
                        n = min(n, max(1, q // int(f2.read().split()[0])))
            break
        except (OSError, ValueError, IndexError):
            continue
    return max(1, min(n, cap))


class CpuPath:
    """The oracle's restatement of the reference path on the host cores (weights and model built once)."""

    def __init__(self, model_name: str, beam: int, sample_tokens: int, seed: int, threads: int, int8: bool = True):
        import torch

        from faster_whisper_b200.config import MODEL_DIMS, special_tokens
        from faster_whisper_b200.synthetic import make_weights, synthetic_audio
        from oracle.whisper_oracle import WhisperOracle

        torch.set_num_threads(threads)
        self.threads, self.beam, self.sample_tokens = threads, beam, sample_tokens
        self.dims = MODEL_DIMS[model_name]
        self.st = special_tokens(self.dims.n_vocab)
        self.int8 = int8
        try:
            self.orc = WhisperOracle(self.dims.to_dict(), make_weights(self.dims, seed=seed), self.st.to_dict(), int8_dynamic=int8)
        except Exception:  # noqa: BLE001 - no quantised engine in this torch build: fall back to fp32 and say so
            self.int8 = False
            self.orc = WhisperOracle(self.dims.to_dict(), make_weights(self.dims, seed=seed), self.st.to_dict())
        self.audio = synthetic_audio(0, 30.0)

    def run(self):
        from oracle.whisper_oracle import log_mel, pad_or_trim

        st, dims, beam, sample_tokens = self.st, self.dims, self.beam, self.sample_tokens
        t0 = time.perf_counter()
        feats = pad_or_trim(log_mel(self.audio, dims.n_mels)[:, :-1])[None]
        t1 = time.perf_counter()
        enc = self.orc.encode(feats)
        t2 = time.perf_counter()
        prompt = [st.sot, st.lang_begin, st.transcribe, st.no_timestamps] if dims.is_multilingual else [st.sot, st.no_timestamps]
        sup = [st.eot, st.sot, st.transcribe, st.translate, st.sot_prev, st.sot_lm, st.no_speech]
        self.orc.generate(enc, [prompt], beam_size=beam, max_length=len(prompt) + sample_tokens, suppress_tokens=sup)
        t3 = time.perf_counter()
        per_tok = (t3 - t2) / (sample_tokens + len(prompt) - 1)
        total = (t1 - t0) + (t2 - t1) + per_tok * (NEW_TOKENS + len(prompt) - 1)
        prec = "dynamic-int8 linears (torch.ao, per-tensor weights)" if self.int8 else "fp32"
        return dict(value=30.0 / total, unit="audio-s/s", cores=self.threads, kind="port", host_cores_available=os.cpu_count(),
                    precision="int8" if self.int8 else "f32",
                    sample=(f"1 chunk of 30 s: log-mel {1e3 * (t1 - t0):.0f} ms + encoder {1e3 * (t2 - t1):.0f} ms measured in full; beam-{beam} "
                            f"decode measured for {sample_tokens} new tokens ({1e3 * per_tok:.0f} ms/position) and scaled to {NEW_TOKENS}; "
                            f"torch CPU restatement of the reference path with {prec} on {self.threads} threads — an approximation of the "
                            "reference's CTranslate2 int8 CPU path, which cannot be installed here"))


def cpu_baseline(model_name: str, beam: int, sample_tokens: int, seed: int, threads: int, int8: bool = True):
    return CpuPath(model_name, beam, sample_tokens, seed, threads, int8).run()


def run_reference(args):
    rank, _, world = dist_env()
    if rank != 0:
        return
    threads = host_threads()
    t0 = time.perf_counter()
    path = CpuPath(args.model, args.beam_size, args.cpu_sample_tokens, args.seed, threads, args.cpu_precision == "int8")
    for _ in range(min(args.warmup, 1)):
        path.run()
    vals = []
    cb = None
    # every step is the same bounded sample (one 30 s chunk, short decode extrapolated); at most 3 are timed so the arm ends in minutes
    for _ in range(max(1, min(args.steps, 3))):
        cb = path.run()
        vals.append(cb["value"])
    v = float(np.mean(vals))
    cb["value"] = v
    line = dict(metric=METRIC, value=v, unit="audio-s/s", n_gpus=args.gpus, steps=args.steps, warmup=args.warmup,
                ms_per_step=30.0 / v * 1e3, higher_is_better=True, scaling="weak", vs_baseline=None,
                dtype="int8" if path.int8 else "f32", data="synthetic", impl="reference",
                config={"workload": workload_name(args), "model": args.model, "timed_samples": len(vals),
                        "note": "CPU port of the reference path on rank 0's host cores; one 30 s chunk per step (per-chunk throughput "
                                "does not depend on the batch on the CPU), decode sample scaled to the pinned length"},
                cpu_baseline=cb, e2e={"value": v, "unit": "audio-s/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                wall_s=time.perf_counter() - t0)
    print(json.dumps(line), flush=True)


def workload_name(args, workload=None):
    workload = workload or args.workload
    prec = "fp16" if not args.compute_type.startswith("int8") else "int8 weights (per-channel, fp16 activations)"
    if workload == "single":
        return f"{args.model} {prec} beam_size={args.beam_size}, single 30 s chunk per step, prompt 4 + {NEW_TOKENS} new tokens (configs[1])"
    cfg = "configs[3]" if args.compute_type.startswith("int8") else "configs[2]"
    return (f"{args.model} {prec} beam_size={args.beam_size}, BatchedInferencePipeline batch_size={args.batch_size}, "
            f"{args.batch_size} x 30 s chunks per step, prompt 4 + {NEW_TOKENS} new tokens ({cfg})")


# ----------------------------------------------------------------------------------------------------------------
def run_engine(args):
    rank, local_rank, world = dist_env()
    use_dist = world > 1
    dist = None
    if use_dist:
        import torch
        import torch.distributed as dist

        # NCCL on a real multi-GPU box; B2W_DIST_BACKEND=gloo lets the same code path be exercised with several ranks on one GPU
        backend = os.environ.get("B2W_DIST_BACKEND", "nccl")
        local_rank = local_rank % max(1, torch.cuda.device_count())
        torch.cuda.set_device(local_rank)
        if backend == "nccl":
            dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
        else:
            dist.init_process_group(backend)

    from faster_whisper_b200 import BatchedInferencePipeline, WhisperModel
    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import synthetic_audio

    dims = MODEL_DIMS[args.model]
    st = special_tokens(dims.n_vocab)
    t_load = time.perf_counter()
    model = WhisperModel(args.model, device="cuda", device_index=local_rank, compute_type=args.compute_type, synthetic_seed=args.seed)
    eng = model.model
    t_load = time.perf_counter() - t_load
    pipe = BatchedInferencePipeline(model)
    prompt = [st.sot, st.lang_begin, st.transcribe, st.no_timestamps] if dims.is_multilingual else [st.sot, st.no_timestamps]
    suppress = sorted({st.eot, st.sot, st.transcribe, st.translate, st.sot_prev, st.sot_lm, st.no_speech})
    pk = peaks()

    def barrier():
        eng.sync()
        if use_dist:
            dist.barrier()

    def measure(workload: str, steps: int, warmup: int, sample_clocks: bool, dump_dir=None):
        """One workload: W warm-up steps, K steps through the engine calls, K steps through the public API."""
        B = 1 if workload == "single" else args.batch_size
        chunks = [synthetic_audio(rank * 1000 + i, 30.0) for i in range(B)]
        audio = np.concatenate(chunks)
        clips = [{"start": 30.0 * i, "end": 30.0 * (i + 1)} for i in range(B)]
        walls = []

        last = {}

        def engine_step():
            enc = eng.encode_audio(chunks)
            res = eng.generate(enc, [prompt] * B, beam_size=args.beam_size, max_length=len(prompt) + NEW_TOKENS, suppress_tokens=suppress,
                               return_scores=True, return_no_speech_prob=True)
            assert all(len(r.sequences_ids[0]) == NEW_TOKENS for r in res)
            last["enc"], last["res"] = enc, res
            return res

        def api_step():
            segs, _ = pipe.transcribe(audio, language="en", beam_size=args.beam_size, batch_size=B, vad_filter=False, clip_timestamps=clips,
                                      max_new_tokens=NEW_TOKENS, suppress_tokens=[-1, st.eot], without_timestamps=True)
            n = sum(len(s.tokens) for s in segs)
            assert n == NEW_TOKENS * B, n
            return n

        def timed(fn):
            """K steps between barrier + sync on both sides, timed on the device: CUDA events recorded on the engine's stream
            before the first and after the last step (host work between launches is inside the span); max over ranks."""
            barrier()
            t0 = time.perf_counter()
            eng.span_begin()
            for _ in range(steps):
                fn()
            dt = eng.span_end() * 1e-3
            eng.sync()
            wall = time.perf_counter() - t0
            if use_dist:
                import torch

                t = torch.tensor([dt, wall], device="cuda" if dist.get_backend() == "nccl" else "cpu")
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                dt, wall = float(t[0].item()), float(t[1].item())
            walls.append(wall)
            return dt

        for _ in range(max(warmup, 3)):
            engine_step()
        api_step()
        eng.timing(enable=True, reset=True)
        sampler = ClockSampler(local_rank) if sample_clocks else None
        if sampler:
            sampler.start()
        dt = timed(engine_step)
        stats = eng.timing()
        eng.timing(enable=False)
        if dump_dir and rank == 0:
            dump_outputs(dump_dir, workload, last["enc"], last["res"])
        dt_api = timed(api_step)
        clocks = sampler.stop() if sampler else None

        audio_s = 30.0 * B * steps * world
        R = B * args.beam_size
        dec_ms = stats["decode_ms"]
        steps_dec = max(1, stats["decode_steps"])
        ach = stats["decode_alg_bytes"] / (dec_ms * 1e-3) / 1e9 if dec_ms > 0 else 0.0
        enc_flops = enc_flops_per_chunk(dims) * B * steps
        enc_tf = enc_flops / (stats["encoder_ms"] * 1e-3) / 1e12 if stats["encoder_ms"] > 0 else 0.0
        kernel = "dstep_kernel" if R <= 8 else "bstep_kernel"
        return dict(
            B=B, value=audio_s / dt, e2e_value=audio_s / dt_api, ms_per_step=dt / steps * 1e3, e2e_ms_per_step=dt_api / steps * 1e3,
            rtf=dt / audio_s * world, h2d=int(audio.nbytes), d2h=int(B * (448 * 4 + 16)), launches=int(stats["launches"]), clocks=clocks,
            stages_ms={k[:-3]: round(v / steps, 3) for k, v in stats.items() if k.endswith("_ms") and v > 0},
            device_ms_per_step=round(sum(v for k, v in stats.items() if k.endswith("_ms")) / steps, 3),
            host_wall_ms_per_step=[round(w / steps * 1e3, 3) for w in walls],
            roofline={"bound": "hbm",
                      "kernel": f"decode step = {kernel} (persistent cooperative kernel: weight stream + self/cross attention + logits) + 2 search kernels",
                      "achieved": ach, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": ach / pk["hbm_gbs"], "peak_source": pk["source"],
                      "ms_per_decode_step": dec_ms / steps_dec,
                      "alg_bytes_per_step": stats["decode_alg_bytes"] / steps_dec},
            roofline_encoder={"bound": "tensor", "achieved": enc_tf, "peak": pk["tflops"], "unit": "TFLOP/s", "frac": enc_tf / pk["tflops"],
                              "flops_per_chunk": enc_flops_per_chunk(dims), "ms_per_chunk": stats["encoder_ms"] / (B * steps)})

    m = measure(args.workload, args.steps, args.warmup, True, args.dump_outputs)
    B = m["B"]
    line = dict(
        metric=METRIC, value=m["value"], unit="audio-s/s", n_gpus=world, steps=args.steps, warmup=max(args.warmup, 3),
        ms_per_step=m["ms_per_step"], higher_is_better=True, scaling="weak", vs_baseline=None,
        dtype="int8" if args.compute_type.startswith("int8") else "f16", data="synthetic", rtf=m["rtf"],
        config={"workload": workload_name(args), "model": args.model, "global_batch": B * world, "beam_size": args.beam_size,
                "new_tokens": NEW_TOKENS, "parallelism": f"chunk-parallel replicas x{world}", "compute_type": args.compute_type,
                "l2": "working set per step (3.1 GB weights + 0.25 GB/chunk cross-KV) exceeds the 50 MB L2; no flush needed",
                "weights": f"synthetic seed {args.seed}, exact {args.model} shapes", "load_s": round(t_load, 1)},
        e2e={"value": m["e2e_value"], "unit": "audio-s/s", "h2d_bytes_per_step": m["h2d"], "d2h_bytes_per_step": m["d2h"],
             "api": "BatchedInferencePipeline.transcribe(ndarray, clip_timestamps=..., batch_size=%d)" % B, "ms_per_step": m["e2e_ms_per_step"]},
        gpu_launches=m["launches"], clocks=m["clocks"], stages_ms=m["stages_ms"], device_ms_per_step=m["device_ms_per_step"],
        timing="value/e2e: CUDA events on the engine stream around the K steps (barrier + sync on both sides, max over ranks); stages_ms/roofline: per-stage CUDA events on the same stream",
        host_wall_ms_per_step=m["host_wall_ms_per_step"], roofline=m["roofline"], roofline_encoder=m["roofline_encoder"],
    )
    if args.workload == "batched" and not args.no_secondary:
        # configs[1] measured in the same process, so both configurations are driver-measured in one line
        s1 = measure("single", args.steps, args.warmup, False)
        line["single_chunk"] = {"workload": workload_name(args, "single"), "value": s1["value"], "unit": "audio-s/s", "ms_per_step": s1["ms_per_step"],
                                "e2e": {"value": s1["e2e_value"], "unit": "audio-s/s", "ms_per_step": s1["e2e_ms_per_step"]},
                                "stages_ms": s1["stages_ms"], "roofline": s1["roofline"], "roofline_encoder": s1["roofline_encoder"]}
    if rank == 0 and world == 1 and not args.no_cpu_baseline:  # reported at N=1 only (the other ranks would idle at the barrier)
        try:
            line["cpu_baseline"] = cpu_baseline(args.model, args.beam_size, args.cpu_sample_tokens, args.seed, host_threads(), args.cpu_precision == "int8")
        except Exception as e:  # noqa: BLE001
            line["cpu_baseline"] = {"value": None, "unit": "audio-s/s", "cores": os.cpu_count(), "kind": "port", "sample": f"failed: {e}"}
    if use_dist:
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(line), flush=True)


def dump_outputs(d: str, workload: str, enc, res) -> None:
    """The arrays a caller of the timed path receives from its last step, as float32 / float64 .npy files (under 64 MB in all)."""
    os.makedirs(d, exist_ok=True)
    np.save(os.path.join(d, f"{workload}_tokens.npy"), np.asarray([r.sequences_ids[0] for r in res], dtype=np.float64))
    np.save(os.path.join(d, f"{workload}_scores.npy"), np.asarray([r.scores[0] for r in res], dtype=np.float64))
    np.save(os.path.join(d, f"{workload}_no_speech_prob.npy"), np.asarray([r.no_speech_prob for r in res], dtype=np.float64))
    e = np.asarray(enc.numpy(), dtype=np.float32).reshape(-1)
    n = min(e.size, 1 << 22)  # 16 MB of float32
    idx = np.sort(np.random.default_rng(1234).integers(0, e.size, n)) if n < e.size else np.arange(e.size)
    np.save(os.path.join(d, f"{workload}_encoder_output_sample.npy"), e[idx])


def enc_flops_per_chunk(dims) -> float:
    d, L, m = dims.n_audio_state, dims.n_audio_layer, dims.n_mels
    lin = 2.0 * (3000 * 3 * m * d + 1500 * 3 * d * d + L * 1500 * (4 * d * d + 2 * d * 4 * d))
    att = L * 4.0 * 1500 * 1500 * d
    return lin + att


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="batched", choices=["single", "batched"])
    ap.add_argument("--compute-type", default="float16", choices=["float16", "int8_float16", "int8"])
    ap.add_argument("--no-secondary", action="store_true", help="skip the single-chunk measurement that rides along with the batched line")
    ap.add_argument("--cpu-precision", default="int8", choices=["int8", "fp32"])
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--beam-size", type=int, default=5)
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--cpu-sample-tokens", type=int, default=32)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the timed path computed in its last step as DIR/<name>.npy (float32 / float64)")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_engine(args)


if __name__ == "__main__":
    main()
