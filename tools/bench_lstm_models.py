"""Throughput of the CaMN (batch 64) and DisCo (batch 32) paths, BASELINE configs[2], [3]: emitted 15-fps frames per
second for 10 s clips, CUDA-event timed (eager launches), next to the CPU oracle on a bounded sample.  JSON lines, each
with the card record."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from synthetic_models import build_lstm_product  # noqa: E402
from oracle import lstm_oracle as L  # noqa: E402
from oracle.weights import make_lstm_checkpoint, synth_audio  # noqa: E402
from pantomatrix_b200.emage_audio import engine  # noqa: E402
from measure import card, mean_ms  # noqa: E402


def main():
    torch.set_num_threads(min(16, os.cpu_count()))
    dev = card()
    for kind, bs in (("camn", 64), ("disco", 32)):
        model = build_lstm_product(kind)
        audio = torch.from_numpy(synth_audio(bs, 160000, 7)).cuda()
        spk = torch.zeros(bs, 1, dtype=torch.long, device="cuda")
        for _ in range(3):
            out = model(audio, spk)
        torch.cuda.synchronize()
        ms = mean_ms(lambda: model(audio, spk), 5)
        frames = bs * out["motion"].shape[1]
        sd, cfg = make_lstm_checkpoint(kind, 0)
        a8 = torch.from_numpy(synth_audio(8, 160000, 7))
        fwd = L.camn_forward if kind == "camn" else L.disco_forward
        with torch.no_grad():
            fwd(sd, cfg, a8[:2], torch.zeros(2, 1, dtype=torch.long))
            t0 = time.perf_counter()
            fwd(sd, cfg, a8, torch.zeros(8, 1, dtype=torch.long))
            cpu_s = time.perf_counter() - t0
        print(json.dumps({"card": dev, "model": kind, "batch": bs, "frames_per_clip": int(out["motion"].shape[1]), "precision": engine.get_precision(),
                          "ms_per_batch": ms, "frames_per_s_15fps": frames / ms * 1e3,
                          "cpu_oracle_frames_per_s": 8 * out["motion"].shape[1] / cpu_s, "cpu_threads": torch.get_num_threads()}))


if __name__ == "__main__":
    main()
