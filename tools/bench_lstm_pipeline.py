"""CaMN / DisCo: eager forward() against the CUDA-graph replay of CapturedLstmPipeline, arms alternating step by step.

    python tools/bench_lstm_pipeline.py OUT_DIR [--steps 20]

  step      CaMN at batch 64 and 1, DisCo at batch 32 and 1, 10 s clips at 16 kHz float32 already on the device:
            model(audio, speaker_id) against pipe(audio).  CUDA events around each step, 256 MB L2 flush before it.
  e2e       CaMN at batch 64 from pinned 48 kHz int16 stereo: CapturedLstmPipeline(input_rate=48000, input_channels=2,
            input_dtype=int16) against the host reader's resample_poly (audio_io.load_audio's host path) followed by
            eager forward().  Same events, so the host resampling is inside the timed span.
  device    torch.cuda.get_device_name and nvidia-smi's name / power.limit, read in the same run.
Medians over --steps; frames are 15-fps output frames.  Writes OUT_DIR/lstm_pipeline.json and prints it."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
SECONDS = 10


def _timed(arms, steps):
    """{name: fn}: every step runs each arm once, in turn, after an L2 flush; returns medians in ms."""
    import torch
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # > the 50 MB L2
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for i in range(steps):
        for k, fn in arms.items():
            flush.fill_(i & 0xFF)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            times[k].append(s.elapsed_time(e))
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}, times


def step_arms(steps):
    import torch
    from oracle.weights import synth_audio
    from pantomatrix_b200.lstm_audio.modeling import wav_frames
    from pantomatrix_b200.pipeline import CapturedLstmPipeline
    from synthetic_models import build_lstm_product
    res = {}
    n = 16000 * SECONDS
    t = wav_frames(n)
    for kind, batches in (("camn", (64, 1)), ("disco", (32, 1))):
        model = build_lstm_product(kind)
        for bs in batches:
            audio = torch.from_numpy(synth_audio(bs, n, 7)).cuda()
            spk = torch.zeros(bs, 1, dtype=torch.long, device="cuda")
            pipe = CapturedLstmPipeline(model, bs, n)
            med, runs = _timed({"eager": lambda: model(audio, spk), "captured": lambda: pipe(audio, spk)}, steps)
            res[f"{kind} batch {bs}"] = {
                "eager_ms": med["eager"], "captured_ms": med["captured"], "speedup": med["eager"] / med["captured"],
                "eager_frames_per_s": bs * t / med["eager"] * 1e3, "captured_frames_per_s": bs * t / med["captured"] * 1e3,
                "kernels_per_replay": pipe.kernels_per_replay, "frames_per_clip": t,
                "runs_ms": {k: [round(x, 3) for x in v] for k, v in runs.items()}}
            del pipe
        del model
        torch.cuda.empty_cache()
    return res


def e2e(steps, bs=64):
    import torch
    from bench_audio_frontend import _host_front_end, _pcm
    from pantomatrix_b200.lstm_audio.modeling import wav_frames
    from pantomatrix_b200.pipeline import CapturedLstmPipeline
    from synthetic_models import build_lstm_product
    model = build_lstm_product("camn")
    pcm = _pcm(bs, 48000, 2, "int16", 7)
    pinned = torch.from_numpy(pcm).pin_memory()
    staging = torch.empty(bs, 16000 * SECONDS).pin_memory()
    spk = torch.zeros(bs, 1, dtype=torch.long, device="cuda")
    pipe = CapturedLstmPipeline(model, bs, pcm.shape[1], input_rate=48000, input_channels=2, input_dtype=torch.int16)
    t = wav_frames(16000 * SECONDS)

    def host_then_eager():
        staging.copy_(torch.from_numpy(_host_front_end(pcm, 48000)))
        model(staging.cuda(non_blocking=True), spk)

    med, runs = _timed({"captured_48k_int16_stereo": lambda: pipe(pinned, spk), "host_resample_then_eager": host_then_eager},
                       steps)
    return {"model": "camn", "batch": bs, **{f"{k}_ms": v for k, v in med.items()},
            **{f"{k}_frames_per_s": bs * t / v * 1e3 for k, v in med.items()},
            "speedup": med["host_resample_then_eager"] / med["captured_48k_int16_stereo"],
            "runs_ms": {k: [round(x, 3) for x in v] for k, v in runs.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_lstm_pipeline.py needs a CUDA device")
    from bench_audio_frontend import device_info
    from pantomatrix_b200.emage_audio import engine
    os.makedirs(args.out_dir, exist_ok=True)
    res = {"device": device_info(), "precision": engine.get_precision(), "seconds_per_clip": SECONDS,
           "timer": "CUDA events around each step, 256 MB L2 flush before it (outside the events), arms alternating, medians",
           "step": step_arms(args.steps), "e2e": e2e(max(3, args.steps // 4))}
    res["device_after"] = device_info()
    with open(os.path.join(args.out_dir, "lstm_pipeline.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
