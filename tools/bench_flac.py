#!/usr/bin/env python
"""FLAC encoding of recorded samples on one GPU (pantomatrix_b200/flac.py), and what an audio track adds to write_mp4.

    python tools/bench_flac.py OUT.json [--reps 5] [--stage-reps 3]

Inputs: speech-like int16 clips (three tones under a slow envelope, plus Gaussian noise; seeded) of 28 s: 16 kHz mono
(the rate the EMAGE front-end reads), 48 kHz stereo (a recorded WAV), and a batch of 8 48 kHz stereo clips.
Reported per input, from CUDA events after a warm-up call (medians over --reps): the flac.encode call (ms), each of
its launches (memset, analyse, emit) timed one by one, and the coded size as a fraction of the raw samples.
Then the output stage for 300 rendered frames (render_body of a seeded pose sequence, 480 x 720, 30 fps) on the host
clock, alternating the arms, medians over --stage-reps: video.write_mp4 without audio, and with the 48 kHz stereo clip
(trimmed to the video's 10 s), into a temporary directory removed after.  The card's name, power limit and max SM
clock are read in the same run.  Nothing is written except OUT."""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from measure import card, event_ms, launch_ms  # noqa: E402
from pantomatrix_b200 import _lib, flac, ops, video  # noqa: E402
from pantomatrix_b200.body_model import SmplxBodyModel  # noqa: E402
from pantomatrix_b200.render import MeshRenderer  # noqa: E402
from synthetic_models import smplx_surface_arrays  # noqa: E402

SECONDS = 28


def speech(n, rate, channels, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    out = []
    for c in range(channels):
        x = sum(a * np.sin(2 * np.pi * f * (1 + 0.01 * c) * t + ph)
                for a, f, ph in ((6000, 180, 0.3), (3000, 450, 1.1), (1500, 1230, 2)))
        out.append(x * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + rng.normal(0, 200, n))
    return np.clip(np.round(np.stack(out, 1)), -32768, 32767).astype(np.int16)


def arm(pcm, rate, reps):
    b, n, c = pcm.shape
    f = flac.frames_of(n)
    data = torch.empty(b * f, flac.slot_bytes(c, 16), dtype=torch.uint8, device="cuda")
    nbytes = torch.empty(b * f, dtype=torch.int64, device="cuda")
    flac.encode(pcm, rate, out=(data, nbytes))                  # warm-up
    torch.cuda.synchronize()
    ms = [event_ms(lambda: flac.encode(pcm, rate, out=(data, nbytes))) for _ in range(reps)]
    coded = int(nbytes.sum())
    rec = torch.empty(b * f * (4 if c == 2 else c), flac.REC_WORDS, dtype=torch.int32, device="cuda")
    st, cs = ops._stream(), n * c
    calls = {
        "memset": lambda: _lib.call("pm_memset_async", data.data_ptr(), 0, data.numel(), st),
        "analyse": lambda: _lib.call("pm_flac_analyse", pcm.data_ptr(), cs, b, n, c, 16, rec.data_ptr(), st),
        "emit": lambda: _lib.call("pm_flac_emit", pcm.data_ptr(), cs, b, n, c, 16, rate, rec.data_ptr(),
                                  data.data_ptr(), data.shape[1], nbytes.data_ptr(), st),
    }
    return {"clips": b, "samples": n, "channels": c, "rate": rate, "frames": b * f,
            "encode_ms_median": statistics.median(ms), "encode_ms_all": ms,
            "stage_ms_median": launch_ms(calls, reps),
            "coded_bytes": coded, "raw_bytes": b * n * c * 2, "coded_fraction_of_raw": coded / (b * n * c * 2)}


def output_stage(frames, pcm, rate, reps):
    res = {"mp4_silent": [], "mp4_with_audio": []}
    size = {}
    for _ in range(reps):
        for name in res:
            d = tempfile.mkdtemp()
            try:
                path = os.path.join(d, "clip.mp4")
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                video.write_mp4(frames, path, fps=30, audio=None if name == "mp4_silent" else (pcm, rate))
                res[name].append(time.perf_counter() - t0)
                size[name] = os.path.getsize(path)
            finally:
                shutil.rmtree(d)
    out = {k: {"s_median": statistics.median(v), "s_all": v, "file_bytes": size[k]} for k, v in res.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stage-reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the FLAC benchmark measures the GPU: no CUDA device found"
    torch.cuda.set_device(0)
    res = {"card": card()}
    mono = torch.as_tensor(speech(16000 * SECONDS, 16000, 1, 0), device="cuda")[None]
    stereo = torch.as_tensor(np.stack([speech(48000 * SECONDS, 48000, 2, s) for s in range(8)]), device="cuda")
    for name, pcm, rate in (("mono_16k_1x28s", mono, 16000), ("stereo_48k_1x28s", stereo[:1], 48000),
                            ("stereo_48k_8x28s", stereo, 48000)):
        res[name] = arm(pcm, rate, args.reps)
        print(name, json.dumps(res[name]), flush=True)
    r = MeshRenderer(SmplxBodyModel(smplx_surface_arrays(), "cuda"))
    t = torch.arange(300, device="cuda", dtype=torch.float32)[:, None]
    poses = torch.zeros(1, 300, 165, device="cuda")
    poses[0, :, 3:66] = 0.2 * torch.sin(t / 20 + torch.arange(63, device="cuda") / 7)
    frames = r.render_body(poses, torch.zeros(1, 300, 3, device="cuda"))[0]
    res["write_mp4_300_frames"] = output_stage(frames, stereo[0], 48000, args.stage_reps)
    print("write_mp4", json.dumps(res["write_mp4_300_frames"]), flush=True)
    res["card_after"] = card()
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
