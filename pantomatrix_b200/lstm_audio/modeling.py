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

    def __call__(self, x):
        for proj, whh in self.layers:
            x = ops.lstm_bidir(proj(x), whh, self.barrier, self.hidden)
        H = self.hidden
        return ops.add2(x[:, :, :H].contiguous(), x[:, :, H:].contiguous())          # forward + backward, C.py:265


class _LstmEngineBase:
    def __init__(self, sd, cfg):
        self.cfg, self.device = cfg, sd["speaker_embedding.weight"].device
        blocks = tuple((stride, pad, stride != 1 or cin != cout) for cin, cout, stride, pad in _BLOCKS)
        self.wav = E._WavEncoder(sd, "audio_encoder", blocks)
        self.spk = sd["speaker_embedding.weight"].contiguous()
        mask = MASK_DICT[cfg["joint_mask"]]
        slot, k = [], 0
        for m in mask:
            slot.append(k if m else -1)
            k += int(m)
        self.n_sel = k
        self.slot = torch.tensor(slot, dtype=torch.int32, device=self.device)

    def features(self, audio, speaker_id, seed_frames, seed_motion):
        """WavEncoder features, speaker rows and the seed-motion block (C.py:238-263): the last two are tiny
        index/fill operations kept in torch (memory plumbing, no arithmetic)."""
        dev = self.device
        audio = audio.to(device=dev, dtype=torch.float32).contiguous()
        a = E._f32(self.wav(audio, 0, 0, 1, audio.shape[1]))
        bs, t, _ = a.shape
        spk = ops.gather_rows(self.spk, speaker_id.to(dev).reshape(-1).to(torch.int64).contiguous()).unsqueeze(1).expand(bs, t, -1)
        dims = int(self.cfg["pose_dims"]) + 1
        if seed_motion is None:
            seed = torch.zeros(bs, t, dims, device=dev)
            seed[:, :seed_frames, -1] = 1
        else:
            t_m = seed_motion.shape[1]
            seed = torch.zeros(bs, t_m, dims, device=dev)
            seed[:, :seed_frames, :-1] = seed_motion.to(dev)[:, :seed_frames]
            seed[:, :seed_frames, -1] = 1
            if t_m > t:
                seed = seed[:, :t]
            elif t_m < t:
                seed = torch.cat((seed, seed[:, -(t - t_m):]), 1)
        return a, spk, seed, bs, t

    def axis_angle(self, motion, bs, t):
        return ops.rot6d_to_aa(motion.reshape(bs, t, self.n_sel * 6).contiguous(), self.slot, self.n_sel)


class _CamnEngine(_LstmEngineBase):
    def __init__(self, sd, cfg):
        super().__init__(sd, cfg)
        H, L = int(cfg["hidden_size"]), int(cfg["n_layer"])
        self.body, self.hands = _BiLstm(sd, "body_motion_decoder", L, H), _BiLstm(sd, "hands_motion_decoder", L, H)
        self.body_out, self.hands_out = E._MLP(sd, "body_out"), E._MLP(sd, "hands_out")

    def forward(self, audio, speaker_id, seed_frames, seed_motion, return_axis_angle):
        a, spk, seed, bs, t = self.features(audio, speaker_id, seed_frames, seed_motion)
        in_fea = torch.cat((a, spk, seed), dim=2)
        body = self.body_out(self.body(in_fea))
        hands = self.hands_out(self.hands(torch.cat((in_fea, body), dim=2)))
        motion = torch.cat((body, hands), dim=2).reshape(bs, t, self.n_sel, 6)          # recombine, C.py:227-234
        return {"motion": motion, "motion_axis_angle": self.axis_angle(motion, bs, t) if return_axis_angle else None}


class _DiscoEngine(_LstmEngineBase):
    def __init__(self, sd, cfg):
        super().__init__(sd, cfg)
        H, L = int(cfg["hidden_size"]), int(cfg["n_layer"])
        self.c1, self.c2, self.r = E._MLP(sd, "audio_encoder_c1"), E._MLP(sd, "audio_encoder_c2"), E._MLP(sd, "audio_encoder_r")
        self.selector = E._MLP(sd, "selector")
        self.body, self.body_out = _BiLstm(sd, "body_motion_decoder", L, H), E._MLP(sd, "body_out")

    def forward(self, audio, speaker_id, seed_frames, seed_motion, return_axis_angle):
        a, spk, seed, bs, t = self.features(audio, speaker_id, seed_frames, seed_motion)
        a = a.contiguous()
        fea_c = ops.softmax2_mix(self.selector(a), self.c1(a), self.c2(a))              # D.py:246-251
        fea_r = self.r(a)
        in_fea = torch.cat((fea_c, fea_r, spk, seed), dim=2)
        motion = self.body_out(self.body(in_fea))
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
        from ..emage_audio import engine as E
        return E.guarded(lambda: self._eng().forward(audio, speaker_id, seed_frames, seed_motion, return_axis_angle),
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
