"""CaMN and DisCo audio->motion models on the H100 path (BASELINE configs[2], [3]).

Same names, forward() signature, outputs, `.cfg` and checkpoint layout as
  C.py = /root/reference/models/camn_audio/modeling_camn_audio.py  (CamnAudioModel, forward 237-281)
  D.py = /root/reference/models/disco_audio/modeling_disco_audio.py (DiscoAudioModel, forward 220-267)
The modules only own parameters; arithmetic runs in libpm_emage.so: WavEncoder convs / Linears as tap-GEMMs (same
engine and precision switch as EMAGE), the LSTM recurrence in the persistent pm_lstm_bidir_f32 kernel, rot6d ->
axis-angle + joint scatter in pm_rot6d_to_aa_f32.  No CPU / eager fallback.
"""
from __future__ import annotations

import torch
from transformers import PretrainedConfig

from .. import ops
from ..emage_audio import engine as E
from ..emage_audio.configuration import _splat
from ..emage_audio import modeling as _M
from ..emage_audio.modeling import _bn, _conv, _EngineOwner, _materialise, _mlp, _plain_state

# (cin, cout, stride, first padding) of the six BasicBlocks, C.py:138-145; a block has a downsample branch iff
# stride != 1 or cin != cout (C.py:113-118)
_BLOCKS = ((1, 32, 5, 1600), (32, 32, 6, 0), (32, 32, 1, 7), (32, 64, 6, 0), (64, 64, 1, 7), (64, 128, 6, 0))
_LOCAL_UPPER = [j in (3, 6, 9) or 12 <= j <= 21 or j >= 25 for j in range(55)]              # C.py:20-27
MASK_DICT = {"local_upper": _LOCAL_UPPER, "local_full": [False] + [True] * 54}


class CamnAudioConfig(PretrainedConfig):
    model_type = "camn_audio"

    def __init__(self, config_obj=None, **kwargs):
        super().__init__(**_splat(config_obj, kwargs))


class DiscoAudioConfig(PretrainedConfig):
    model_type = "disco_audio"

    def __init__(self, config_obj=None, **kwargs):
        super().__init__(**_splat(config_obj, kwargs))


def _wav_spec(p):
    s = []
    for i, (cin, cout, stride, _) in enumerate(_BLOCKS):
        q = f"{p}.feat_extractor.{i}"
        s += _conv(q + ".conv1", cout, cin, 15) + _bn(q + ".bn1", cout) + _conv(q + ".conv2", cout, cout, 15) + _bn(q + ".bn2", cout)
        if stride != 1 or cin != cout:
            s += _conv(q + ".downsample.0", cout, cin, 15) + _bn(q + ".downsample.1", cout)
    return s


def _lstm_spec(p, in_dim, hidden, n_layer):
    s = []
    for layer in range(n_layer):
        d = in_dim if layer == 0 else 2 * hidden
        for suffix in ("", "_reverse"):
            s += [(f"{p}.weight_ih_l{layer}{suffix}", (4 * hidden, d), "p"), (f"{p}.weight_hh_l{layer}{suffix}", (4 * hidden, hidden), "p"),
                  (f"{p}.bias_ih_l{layer}{suffix}", (4 * hidden,), "p"), (f"{p}.bias_hh_l{layer}{suffix}", (4 * hidden,), "p")]
    return s


class _BiLstm:
    """Packed nn.LSTM(batch_first, bidirectional): per layer one input-projection GEMM for both directions and all
    time steps (N = 8H) + the persistent recurrent kernel."""

    def __init__(self, sd, p, n_layer, hidden):
        self.hidden, self.layers = hidden, []
        for layer in range(n_layer):
            w = torch.cat([sd[f"{p}.weight_ih_l{layer}"], sd[f"{p}.weight_ih_l{layer}_reverse"]], 0)
            b = torch.cat([sd[f"{p}.bias_ih_l{layer}"] + sd[f"{p}.bias_hh_l{layer}"],
                           sd[f"{p}.bias_ih_l{layer}_reverse"] + sd[f"{p}.bias_hh_l{layer}_reverse"]], 0)
            whh = torch.stack([sd[f"{p}.weight_hh_l{layer}"], sd[f"{p}.weight_hh_l{layer}_reverse"]], 0).contiguous()
            self.layers.append((E._Linear(None, w=w, b=b), whh))
        self.barrier = torch.zeros(4, dtype=torch.int32, device=sd[f"{p}.weight_hh_l0"].device)

    def __call__(self, x, barrier=None):
        """barrier: int32[4] device scratch of the recurrent kernel (default: this stack's own).  A caller that runs the
        stack on another stream than the default owner - a captured graph - passes its own."""
        barrier = self.barrier if barrier is None else barrier
        for proj, whh in self.layers:
            x = ops.lstm_bidir(proj(x), whh, barrier, self.hidden)
        H = self.hidden
        return ops.add2(x[:, :, :H], x[:, :, H:])             # forward + backward, C.py:265, halves read in place


def wav_frames(n: int) -> int:
    """Frames the CaMN / DisCo WavEncoder emits for n samples (C.py:138-145 conv arithmetic)."""
    for _, _, stride, pad in _BLOCKS:
        n = (n + 2 * pad - 15) // stride + 1
    return n


def _round4(n):
    return (n + 3) // 4 * 4


def _mlp_into(mlp, x, *outs):
    """MLP (P.py:316-326) whose last Linear writes each of `outs` (fp32 views; None = a new dense tensor): the hidden
    layer runs once, the output GEMM once per target, so no copy kernel is needed to place a result twice."""
    h = mlp.fc1(x, act=ops.ACT_LEAKY, slope=0.1, want="p")
    return [mlp.fc2(h, out=o) for o in outs]


class _LstmEngineBase:
    """The layer-0 LSTM input is one (batch, t, width) buffer, row stride rounded up to 16 bytes, whose column ranges
    are written in place: the audio features by their last GEMM, the conditioning columns (speaker row | seed pose |
    seed flag, C.py:238-263) by a `cond(dest)` filler.  forward() takes the filler, so the step has one schedule:
      host_cond    the eager forward(): the reference's seed handling for any seed tensor, as index / fill operations
                   on the device (memory plumbing, no arithmetic);
      kernel_cond  the captured step (pipeline.CapturedLstmPipeline): one pm_lstm_cond_f32 launch over static buffers,
                   so the graph holds library kernels and memset nodes only."""

    def __init__(self, sd, cfg):
        self.cfg, self.device = cfg, sd["speaker_embedding.weight"].device
        blocks = tuple((stride, pad, stride != 1 or cin != cout) for cin, cout, stride, pad in _BLOCKS)
        self.wav = E._WavEncoder(sd, "audio_encoder", blocks)
        self.wav_dim = _BLOCKS[-1][1]
        self.spk = sd["speaker_embedding.weight"].contiguous()
        self.pose_dims = int(cfg["pose_dims"])
        self.cond_dim = self.spk.shape[1] + self.pose_dims + 1             # speaker row | seed pose | seed flag
        mask = MASK_DICT[cfg["joint_mask"]]
        slot, k = [], 0
        for m in mask:
            slot.append(k if m else -1)
            k += int(m)
        self.n_sel = k
        self.slot = torch.tensor(slot, dtype=torch.int32, device=self.device)

    def host_cond(self, speaker_id, seed_frames, seed_motion):
        """Filler for forward(speaker_id, seed_frames, seed_motion): C.py:238-263 written into the destination view.  A
        seed of t_m rows is cut to t rows or extended by its own last t - t_m rows (defined for t <= 2*t_m); its first
        seed_frames rows (Python slice semantics) carry the flag.  No seed = zeros over t rows."""
        dev, nspk = self.device, self.spk.shape[1]
        ids = speaker_id.to(dev).reshape(-1).to(torch.int64).contiguous()

        def fill(dest):
            t = dest.shape[1]
            dest[:, :, :nspk] = ops.gather_rows(self.spk, ids).unsqueeze(1)
            seed = dest[:, :, nspk:]
            seed.zero_()
            if seed_motion is None:
                seed[:, :seed_frames, -1] = 1
                return
            t_m = seed_motion.shape[1]
            if t > 2 * t_m:
                raise ValueError(f"seed_motion has {t_m} frames; the audio gives {t}, at most twice as many")
            src = seed_motion.to(dev)[:, :seed_frames][:, :t]
            seed[:, :src.shape[1], :-1] = src
            seed[:, :src.shape[1], -1] = 1
            if t_m < t:
                seed[:, t_m:] = seed[:, 2 * t_m - t:t_m]
        return fill

    def kernel_cond(self, speaker_id, seed, seed_len, seed_frames):
        """Filler of the captured step: speaker_id (batch, 1) int64 and seed (batch, >= min(seed_frames, seed_len),
        pose_dims) fp32 device buffers; the seed stands for seed_len rows (pm_lstm_cond_f32 in include/pm_emage.h)."""
        return lambda dest: ops.lstm_cond(self.spk, speaker_id, seed, seed_len, seed_frames, self.pose_dims, dest)

    def audio_frames(self, audio):
        audio = audio.to(device=self.device, dtype=torch.float32).contiguous()
        return audio, audio.shape[0], wav_frames(audio.shape[1])

    def axis_angle(self, motion, bs, t):
        return ops.rot6d_to_aa(motion.reshape(bs, t, self.n_sel * 6), self.slot, self.n_sel)


class _CamnEngine(_LstmEngineBase):
    def __init__(self, sd, cfg):
        super().__init__(sd, cfg)
        H, L = int(cfg["hidden_size"]), int(cfg["n_layer"])
        self.body, self.hands = _BiLstm(sd, "body_motion_decoder", L, H), _BiLstm(sd, "hands_motion_decoder", L, H)
        self.body_out, self.hands_out = E._MLP(sd, "body_out"), E._MLP(sd, "hands_out")
        self.body_dims, self.hands_dims = self.body_out.fc2.w.shape[1], self.hands_out.fc2.w.shape[1]

    def forward(self, audio, cond, return_axis_angle, barrier=None):
        """cond: conditioning filler (host_cond / kernel_cond); barrier: see _BiLstm."""
        audio, bs, t = self.audio_frames(audio)
        c0 = self.wav_dim                                          # hands input: audio | speaker | seed | body
        b0 = c0 + self.cond_dim
        x = torch.empty(bs, t, _round4(b0 + self.body_dims), device=self.device)
        self.wav(audio, 0, 0, 1, audio.shape[1], out=x[:, :, :c0])
        cond(x[:, :, c0:b0])
        motion = torch.empty(bs, t, self.body_dims + self.hands_dims, device=self.device)   # body | hands, C.py:227-234
        _mlp_into(self.body_out, self.body(x[:, :, :b0], barrier), motion[:, :, :self.body_dims],
                  x[:, :, b0:b0 + self.body_dims])
        self.hands_out(self.hands(x[:, :, :b0 + self.body_dims], barrier), out=motion[:, :, self.body_dims:])
        motion = motion.view(bs, t, self.n_sel, 6)
        return {"motion": motion, "motion_axis_angle": self.axis_angle(motion, bs, t) if return_axis_angle else None}


class _DiscoEngine(_LstmEngineBase):
    def __init__(self, sd, cfg):
        super().__init__(sd, cfg)
        H, L = int(cfg["hidden_size"]), int(cfg["n_layer"])
        self.c1, self.c2, self.r = E._MLP(sd, "audio_encoder_c1"), E._MLP(sd, "audio_encoder_c2"), E._MLP(sd, "audio_encoder_r")
        self.selector = E._MLP(sd, "selector")
        self.body, self.body_out = _BiLstm(sd, "body_motion_decoder", L, H), E._MLP(sd, "body_out")
        self.fea_dim = self.r.fc2.w.shape[1]

    def forward(self, audio, cond, return_axis_angle, barrier=None):
        audio, bs, t = self.audio_frames(audio)
        a = self.wav(audio, 0, 0, 1, audio.shape[1])
        f = self.fea_dim                                           # LSTM input: content | rhythm | speaker | seed
        width = 2 * f + self.cond_dim
        x = torch.empty(bs, t, _round4(width), device=self.device)
        sel, c1, c2 = self.selector(a), self.c1(a), self.c2(a)
        fea_c = ops.softmax2_mix(sel, c1, c2)                      # D.py:246-251: the output, and in place in the input
        ops.softmax2_mix(sel, c1, c2, out=x[:, :, :f])
        fea_r, _ = _mlp_into(self.r, a, None, x[:, :, f:2 * f])
        cond(x[:, :, 2 * f:width])
        motion = self.body_out(self.body(x[:, :, :width], barrier))
        aa = self.axis_angle(motion, bs, t) if return_axis_angle else None
        return {"motion": motion, "motion_axis_angle": aa, "audio_fea_c": fea_c, "audio_fea_r": fea_r}


class _LstmModelBase(_EngineOwner):
    _engine_cls = None

    def _eng(self):
        if self._engine is None:
            _M._require_cuda(self, type(self).__name__)
            self._engine = self._engine_cls(_plain_state(self), self.cfg.to_dict())
        return self._engine

    def forward(self, audio, speaker_id, seed_frames=4, seed_motion=None, return_axis_angle=True):
        """audio (bs, n) 16 kHz, speaker_id (bs, 1) long, optional seed_motion (bs, t_m, pose_dims) rot6d."""
        eng = self._eng()
        return E.guarded(lambda: eng.forward(audio, eng.host_cond(speaker_id, seed_frames, seed_motion), return_axis_angle),
                         lambda out: [out["motion"]])


class CamnAudioPreTrainedModel(_LstmModelBase):
    config_class = CamnAudioConfig
    base_model_prefix = "camn_audio"


class CamnAudioModel(CamnAudioPreTrainedModel):
    """C.py:187-281."""
    _engine_cls = _CamnEngine

    def __init__(self, config: CamnAudioConfig):
        super().__init__(config)
        self.cfg, self.pose_rep, self.joint_mask = config, config.pose_rep, MASK_DICT[config.joint_mask]
        if config.pose_rep != "smplx":
            raise NotImplementedError("only the shipped pose_rep='smplx' configuration is on the GPU path")
        H, L = config.hidden_size, config.n_layer
        in_body = config.pose_dims + 1 + config.speaker_f + config.audio_f
        spec = _wav_spec("audio_encoder") + [("speaker_embedding.weight", (config.speaker_dims, config.speaker_f), "p")]
        spec += _lstm_spec("body_motion_decoder", in_body, H, L) + _mlp("body_out", H, H, config.body_dims)
        spec += _lstm_spec("hands_motion_decoder", in_body + config.body_dims, H, L) + _mlp("hands_out", H, H, config.hands_dims)
        _materialise(self, spec)
        self.post_init()


class DiscoAudioPreTrainedModel(_LstmModelBase):
    config_class = DiscoAudioConfig
    base_model_prefix = "camn_audio"          # sic: the reference reuses the CaMN prefix (D.py:177)


class DiscoAudioModel(DiscoAudioPreTrainedModel):
    """D.py:183-267."""
    _engine_cls = _DiscoEngine

    def __init__(self, config: DiscoAudioConfig):
        super().__init__(config)
        self.cfg, self.pose_rep, self.joint_mask = config, config.pose_rep, MASK_DICT[config.joint_mask]
        H, L, af = config.hidden_size, config.n_layer, config.audio_f
        spec = _wav_spec("audio_encoder") + [("speaker_embedding.weight", (config.speaker_dims, config.speaker_f), "p")]
        for n in ("audio_encoder_c1", "audio_encoder_c2", "audio_encoder_r"):
            spec += _mlp(n, af, H, af)
        spec += _mlp("selector", af, H, 2)
        spec += _lstm_spec("body_motion_decoder", config.pose_dims + 1 + config.speaker_f + 2 * af, H, L)
        spec += _mlp("body_out", H, H, config.pose_dims)
        _materialise(self, spec)
        self.post_init()
