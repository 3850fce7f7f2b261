"""Caller plumbing of the hot path: the timed span of the reference demo
(/root/reference/test_emage_audio.py:16-47, twin train_emage_audio.py:33-102) without audio file
decoding and npz writing: inference() -> indices from the concatenated logits -> full-length
decode(get_global_motion=True)."""
from __future__ import annotations

import torch

from . import _lib, ops
from .emage_audio.engine import PARTS, select_inputs

_OVERFLOW = ("fp16x3: a GEMM operand exceeded the fp16 range (|x| > 1023 after the x64 pre-scale) and the result is NaN - "
             "use engine.set_precision('bf16x6') for this checkpoint (model.inference() outside a captured graph retries "
             "in bf16x6 by itself)")


@torch.no_grad()
def generate(model, motion_vq, audio, speaker_id=None, masked_motion=None, mask=None, ref_trans=None):
    """audio (bs, n) float32 16 kHz.  Returns (latent_dict, pred_dict) like T.py:32 and T.py:44-47."""
    dev = next(model.parameters()).device
    bs = audio.shape[0]
    if speaker_id is None:
        speaker_id = torch.zeros(bs, 1, dtype=torch.long, device=dev)                  # T.py:19
    lat = model.inference(audio, speaker_id, motion_vq, masked_motion=masked_motion, mask=mask)
    # fp16 operand planes turn an out-of-range activation into inf - inf = NaN in the consuming GEMM; a NaN anywhere
    # upstream reaches the logits (cls_* = MLP(rec_*)), which the argmax kernels read anyway: they raise the flag.
    generate.nonfinite = ops.zero_flag(dev) if ops.plane_format() == "fp16" else None
    cfg = model.cfg.to_dict()
    idx = {p: ops.row_argmax(lat["cls_" + p], nonfinite=generate.nonfinite) for p in PARTS}       # T.py:39-42
    if generate.nonfinite is not None:
        capturing = lat["rec_face"].is_cuda and torch.cuda.is_current_stream_capturing()
        if not capturing and bool(generate.nonfinite):
            raise _lib.PmError(_OVERFLOW)
    index, latent = select_inputs(cfg, lat, idx)
    if ref_trans is None:
        ref_trans = torch.zeros(1, 3, device=dev)                                       # trans[:,0], T.py:30,47
    pred = motion_vq.decode(
        face_latent=latent["face"], upper_latent=latent["upper"], lower_latent=latent["lower"],
        hands_latent=latent["hands"], face_index=index["face"], upper_index=index["upper"],
        lower_index=index["lower"], hands_index=index["hands"], get_global_motion=True, ref_trans=ref_trans)
    return lat, pred


generate.nonfinite = None


class CapturedPipeline:
    """generate() captured once into a CUDA graph for a fixed (batch, n_samples) and replayed per call.

    The hot path is ~10^3 small kernel launches per step; replaying them as one graph removes the Python /
    launch latency between kernels (launch-bound inner loops belong in CUDA graphs).  Inputs
    are copied into static device buffers, outputs are static tensors owned by this object (valid until
    the next call).  Only the default-input form of the demo (masked_motion=None, mask=None) is captured.
    """

    def __init__(self, model, motion_vq, batch: int, n_samples: int, warmup: int = 2, body_priority: bool = True,
                 input_rate: int = 16000, input_channels: int = 1, input_dtype=torch.float32):
        self.model, self.vq = model, motion_vq
        dev = next(model.parameters()).device
        self.device = dev
        # Recorded audio as it comes (any rate, int16 / float32, 1-8 interleaved channels): a (batch, n_samples,
        # channels) input buffer at input_rate, and the resampling kernel as the first node of the graph, writing the
        # 16 kHz buffer that generate() reads.  The defaults (16 kHz float32 mono) take the audio as it is.
        self.pcm = self.resampler = None
        if (input_rate, input_channels, input_dtype) != (16000, 1, torch.float32):
            from .audio_io import Resampler
            if input_dtype not in (torch.int16, torch.float32) or not 1 <= input_channels <= 8:
                raise ValueError(f"input must be int16 or float32 with 1-8 channels, got {input_dtype} x {input_channels}")
            self.resampler = Resampler(input_rate, 16000, device=dev)
            self.pcm = torch.zeros(batch, n_samples, input_channels, device=dev, dtype=input_dtype)
            self.audio = torch.zeros(batch, self.resampler.n_out(n_samples), device=dev)
        else:
            self.audio = torch.zeros(batch, n_samples, device=dev)
        self.speaker_id = torch.zeros(batch, 1, dtype=torch.long, device=dev)
        self.ref_trans = torch.zeros(1, 3, device=dev)

        def step():
            if self.resampler is not None:
                self.resampler(self.pcm, out=self.audio)
            return generate(model, motion_vq, self.audio, self.speaker_id, ref_trans=self.ref_trans)

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                        # warm-up off the capture: lazy packing, attributes
            for _ in range(warmup):
                step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        before = ops.launch_count
        # The capture stream carries the longest dependency chain (the body stack: 1 + 8 layers per window); the face /
        # refine / part branches fork onto default-priority side streams.  Capturing on a high-priority stream makes the
        # kernel nodes of the critical chain win when both have thread blocks ready (a 96-CTA GEMM leaves 52 SMs free,
        # which the other branch's blocks share).
        self.capture_stream = torch.cuda.Stream(device=dev, priority=-1) if body_priority else None
        with torch.cuda.graph(self.graph, stream=self.capture_stream):
            self.latent, self.pred = step()
        self.kernels_per_replay = ops.launch_count - before
        self.nonfinite = generate.nonfinite                  # fp16 planes only: in-graph overflow flag (else None)

    @torch.no_grad()
    def __call__(self, audio, speaker_id=None):
        """audio: (batch, n_samples) float32, host (pinned for async copies) or device.  With a recorded-audio input
        (input_rate / input_channels / input_dtype): exactly (batch, n_samples, input_channels) of input_dtype, in
        pinned host memory or on this pipeline's device."""
        if self.pcm is None:
            self.audio.copy_(audio, non_blocking=True)
        else:
            want = (tuple(self.pcm.shape), self.pcm.dtype)
            if not torch.is_tensor(audio) or (tuple(audio.shape), audio.dtype) != want:
                got = (tuple(audio.shape), audio.dtype) if torch.is_tensor(audio) else type(audio).__name__
                raise ValueError(f"CapturedPipeline input must be a {want[0]} {want[1]} tensor, got {got}")
            if audio.is_cuda and audio.device != self.pcm.device:
                raise ValueError(f"CapturedPipeline input is on {audio.device}, the pipeline on {self.pcm.device}")
            if not audio.is_cuda and not audio.is_pinned():
                raise ValueError("CapturedPipeline host input must be in pinned memory (tensor.pin_memory())")
            self.pcm.copy_(audio, non_blocking=True)
        if speaker_id is not None:
            self.speaker_id.copy_(speaker_id, non_blocking=True)
        self.graph.replay()
        ops.launch_count += self.kernels_per_replay
        if self.nonfinite is not None and bool(self.nonfinite):     # one 4-byte read back per step (fp16 planes only)
            raise _lib.PmError(_OVERFLOW)
        return self.latent, self.pred
