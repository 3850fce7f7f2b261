"""Caller plumbing of the hot path: the timed span of the reference demo
(/root/reference/test_emage_audio.py:16-47, twin train_emage_audio.py:33-102) without audio file
decoding and npz writing: inference() -> indices from the concatenated logits -> full-length
decode(get_global_motion=True)."""
from __future__ import annotations

import torch

from . import _lib, ops
from .emage_audio.engine import PARTS, overflow_flag, select_inputs

_OVERFLOW = ("fp16x3: a GEMM operand exceeded the fp16 range (|x| > 1023 after the x64 pre-scale) and the result is NaN - "
             "use engine.set_precision('bf16x6') for this checkpoint (model.inference() outside a captured graph retries "
             "in bf16x6 by itself)")


def generate(model, motion_vq, audio, speaker_id=None, masked_motion=None, mask=None, ref_trans=None):
    """audio (bs, n) float32 16 kHz.  Returns (latent_dict, pred_dict) like T.py:32 and T.py:44-47."""
    return _generate(model, motion_vq, audio, speaker_id, masked_motion, mask, ref_trans)[:2]


@torch.no_grad()
def _generate(model, motion_vq, audio, speaker_id=None, masked_motion=None, mask=None, ref_trans=None):
    """generate() -> (latent_dict, pred_dict, the fp16 overflow flag of engine.overflow_flag or None).  Outside a
    graph capture an overflow raises PmError; inside one the caller reads the flag after each replay."""
    dev = next(model.parameters()).device
    bs = audio.shape[0]
    if speaker_id is None:
        speaker_id = torch.zeros(bs, 1, dtype=torch.long, device=dev)                  # T.py:19
    lat = model.inference(audio, speaker_id, motion_vq, masked_motion=masked_motion, mask=mask)
    # a NaN anywhere upstream reaches the logits (cls_* = MLP(rec_*)), which the argmax kernels read anyway
    nonfinite = overflow_flag(dev)
    cfg = model.cfg.to_dict()
    idx = {p: ops.row_argmax(lat["cls_" + p], nonfinite=nonfinite) for p in PARTS}            # T.py:39-42
    if nonfinite is not None:
        capturing = lat["rec_face"].is_cuda and torch.cuda.is_current_stream_capturing()
        if not capturing and bool(nonfinite):
            raise _lib.PmError(_OVERFLOW)
    index, latent = select_inputs(cfg, lat, idx)
    if ref_trans is None:
        ref_trans = torch.zeros(1, 3, device=dev)                                       # trans[:,0], T.py:30,47
    pred = motion_vq.decode(
        face_latent=latent["face"], upper_latent=latent["upper"], lower_latent=latent["lower"],
        hands_latent=latent["hands"], face_index=index["face"], upper_index=index["upper"],
        lower_index=index["lower"], hands_index=index["hands"], get_global_motion=True, ref_trans=ref_trans)
    return lat, pred, nonfinite


def _audio_input(batch, n_samples, dev, input_rate, input_channels, input_dtype):
    """Static audio buffers of a captured pipeline: (pcm, resampler, audio).  Recorded audio as it comes (any rate,
    int16 / float32, 1-8 interleaved channels) lands in a (batch, n_samples, channels) pcm buffer, and the resampling
    kernel - the first node of the graph - writes the 16 kHz buffer the model reads.  The defaults (16 kHz float32 mono)
    take the audio as it is: pcm and resampler are None."""
    if (input_rate, input_channels, input_dtype) == (16000, 1, torch.float32):
        return None, None, torch.zeros(batch, n_samples, device=dev)
    from .audio_io import Resampler
    if input_dtype not in (torch.int16, torch.float32) or not 1 <= input_channels <= 8:
        raise ValueError(f"input must be int16 or float32 with 1-8 channels, got {input_dtype} x {input_channels}")
    resampler = Resampler(input_rate, 16000, device=dev)
    pcm = torch.zeros(batch, n_samples, input_channels, device=dev, dtype=input_dtype)
    return pcm, resampler, torch.zeros(batch, resampler.n_out(n_samples), device=dev)


def _stage(dst, src, who, exact):
    """Copy one call's input into its static buffer (asynchronously).  exact: the input must have the buffer's shape
    and dtype and sit in pinned host memory or on the buffer's device (recorded audio; nothing is converted)."""
    if exact:
        want = (tuple(dst.shape), dst.dtype)
        if not torch.is_tensor(src) or (tuple(src.shape), src.dtype) != want:
            got = (tuple(src.shape), src.dtype) if torch.is_tensor(src) else type(src).__name__
            raise ValueError(f"{who} input must be a {want[0]} {want[1]} tensor, got {got}")
        if src.is_cuda and src.device != dst.device:
            raise ValueError(f"{who} input is on {src.device}, the pipeline on {dst.device}")
        if not src.is_cuda and not src.is_pinned():
            raise ValueError(f"{who} host input must be in pinned memory (tensor.pin_memory())")
    dst.copy_(src, non_blocking=True)


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
        self.pcm, self.resampler, self.audio = _audio_input(batch, n_samples, dev, input_rate, input_channels, input_dtype)
        self.speaker_id = torch.zeros(batch, 1, dtype=torch.long, device=dev)
        self.ref_trans = torch.zeros(1, 3, device=dev)

        def step():
            if self.resampler is not None:
                self.resampler(self.pcm, out=self.audio)
            return _generate(model, motion_vq, self.audio, self.speaker_id, ref_trans=self.ref_trans)

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
            self.latent, self.pred, self.nonfinite = step()   # nonfinite: the in-graph overflow flag (fp16x3 only)
        self.kernels_per_replay = ops.launch_count - before

    @torch.no_grad()
    def __call__(self, audio, speaker_id=None):
        """audio: (batch, n_samples) float32, host (pinned for async copies) or device.  With a recorded-audio input
        (input_rate / input_channels / input_dtype): exactly (batch, n_samples, input_channels) of input_dtype, in
        pinned host memory or on this pipeline's device."""
        if self.pcm is None:
            _stage(self.audio, audio, "CapturedPipeline", exact=False)
        else:
            _stage(self.pcm, audio, "CapturedPipeline", exact=True)
        if speaker_id is not None:
            self.speaker_id.copy_(speaker_id, non_blocking=True)
        self.graph.replay()
        ops.launch_count += self.kernels_per_replay
        if self.nonfinite is not None and bool(self.nonfinite):     # one 4-byte read back per step (fp16 planes only)
            raise _lib.PmError(_OVERFLOW)
        return self.latent, self.pred


def _memset0(t):
    _lib.call("pm_memset_async", t.data_ptr(), 0, t.numel() * t.element_size(), torch.cuda.current_stream(t.device).cuda_stream)


class CapturedLstmPipeline:
    """CaMN / DisCo forward() captured once into a CUDA graph for a fixed (batch, n_samples) and replayed per call.

    model: a CamnAudioModel or DiscoAudioModel.  The graph holds library kernels and memset nodes only: the optional
    resampling of recorded audio (input_rate / input_channels / input_dtype, as in CapturedPipeline), the WavEncoder,
    the in-place assembly of the LSTM inputs, the recurrences and the heads.  Speaker ids and the first seed_frames seed
    poses are static inputs.  The pipeline owns the LSTM barrier scratch, so an eager forward() of the same model on
    another stream cannot interfere with a replay.  The precision mode in effect at construction is the one captured;
    in fp16x3 an in-graph flag turns an operand overflow into PmError after the replay.  Outputs are a static dict with
    the keys of forward(), valid until the next call."""

    def __init__(self, model, batch: int, n_samples: int, seed_frames: int = 4, warmup: int = 2,
                 input_rate: int = 16000, input_channels: int = 1, input_dtype=torch.float32):
        from .lstm_audio.modeling import wav_frames
        if seed_frames < 0:
            raise ValueError(f"seed_frames must be >= 0, got {seed_frames}")
        dev = next(model.parameters()).device
        self.model, self.device, self.batch, self.seed_frames = model, dev, batch, seed_frames
        self.pcm, self.resampler, self.audio = _audio_input(batch, n_samples, dev, input_rate, input_channels, input_dtype)
        eng = model._eng()
        self.speaker_dims, self.pose_dims = eng.spk.shape[0], eng.pose_dims
        self.speaker_id = torch.zeros(batch, 1, dtype=torch.long, device=dev)
        self.seed = torch.zeros(batch, seed_frames, self.pose_dims, device=dev)
        self.barrier = torch.zeros(4, dtype=torch.int32, device=dev)
        t = wav_frames(self.audio.shape[1])

        @torch.no_grad()
        def step():
            if self.resampler is not None:
                self.resampler(self.pcm, out=self.audio)
            # seed_len = t: the seed buffer stands for a t-frame seed whose rows past seed_frames are zeros, which is
            # forward(seed_motion=x) for any x of length t with these first rows (and forward(seed_motion=None) for zeros)
            out = eng.forward(self.audio, eng.kernel_cond(self.speaker_id, self.seed, t, seed_frames), True,
                              barrier=self.barrier)
            flag = overflow_flag(dev)
            if flag is not None:           # an fp16 operand overflow leaves NaN in the motion: the argmax kernel flags it
                ops.row_argmax(out["motion"], nonfinite=flag)
            return out, flag

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                        # warm-up off the capture: lazy packing, attributes
            for _ in range(warmup):
                step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        before = ops.launch_count
        with torch.cuda.graph(self.graph):
            self.out, self.nonfinite = step()
        self.kernels_per_replay = ops.launch_count - before

    def _stage_inputs(self, audio, speaker_id, seed_motion):
        """Validate one call's inputs and copy them into the static buffers (asynchronously)."""
        if self.pcm is None:
            _stage(self.audio, audio, "CapturedLstmPipeline", exact=False)
        else:
            _stage(self.pcm, audio, "CapturedLstmPipeline", exact=True)
        if speaker_id is None:
            _memset0(self.speaker_id)
        else:
            if not torch.is_tensor(speaker_id) or tuple(speaker_id.shape) != (self.batch, 1) or speaker_id.dtype != torch.int64:
                got = (tuple(speaker_id.shape), speaker_id.dtype) if torch.is_tensor(speaker_id) else type(speaker_id).__name__
                raise ValueError(f"speaker_id must be a ({self.batch}, 1) int64 tensor, got {got}")
            lo, hi = int(speaker_id.min()), int(speaker_id.max())
            if lo < 0 or hi >= self.speaker_dims:
                raise ValueError(f"speaker_id must lie in [0, {self.speaker_dims}), got values in [{lo}, {hi}]")
            self.speaker_id.copy_(speaker_id, non_blocking=True)
        if seed_motion is None:
            _memset0(self.seed)
        else:
            want = (self.batch, self.seed_frames, self.pose_dims)
            if not torch.is_tensor(seed_motion) or tuple(seed_motion.shape) != want or seed_motion.dtype != torch.float32:
                got = (tuple(seed_motion.shape), seed_motion.dtype) if torch.is_tensor(seed_motion) else type(seed_motion).__name__
                raise ValueError(f"seed_motion must be a {want} float32 tensor or None, got {got}")
            self.seed.copy_(seed_motion, non_blocking=True)

    @torch.no_grad()
    def __call__(self, audio, speaker_id=None, seed_motion=None):
        """audio as for CapturedPipeline; speaker_id (batch, 1) int64 in [0, speaker_dims), None = zeros; seed_motion
        (batch, seed_frames, pose_dims) float32 rot6d of the first frames, None = zeros (= forward(seed_motion=None))."""
        self._stage_inputs(audio, speaker_id, seed_motion)
        self.graph.replay()
        ops.launch_count += self.kernels_per_replay
        if self.nonfinite is not None and bool(self.nonfinite):     # one 4-byte read back per step (fp16 planes only)
            raise _lib.PmError(_OVERFLOW)
        return self.out
