"""Drop-in replacements for the reference's `models.emage_audio` modules on H100.

Same class names, constructor / forward() / inference() / decode() signatures, `.cfg` attributes,
Hugging Face checkpoint layout (state_dict keys, config.json + model.safetensors) and error behaviour
as /root/reference/models/emage_audio/modeling_emage_audio.py (M.py) - but the modules own only the
parameters; all arithmetic runs in the sm_90a kernels of libpm_emage.so through `engine.py`.

There is deliberately NO CPU or PyTorch-eager path: calling forward()/inference()/decode() with the
module on a non-CUDA device, or without the built library, raises.
"""
from __future__ import annotations

import torch
import torch.nn as nn
from transformers import PreTrainedModel

from .. import _lib, ops
from . import engine as E
from .configuration import EmageAudioConfig, EmageVAEConvConfig, EmageVQVAEConvConfig

# ----------------------------------------------------------------------------------------------------
# Parameter containers.  The checkpoint layout is described as a flat list of (key, shape, kind) and
# materialised as nested bare nn.Modules, so state_dict() keys equal the reference's without mirroring
# its module classes.  kind: "p" parameter, "b" float buffer, "n" int64 scalar buffer.
# ----------------------------------------------------------------------------------------------------


class _Holder(nn.Module):
    """A node of the checkpoint tree: parameters/buffers only, no forward."""


def _materialise(root: nn.Module, spec):
    for key, shape, kind in spec:
        node = root
        *path, leaf = key.split(".")
        for name in path:
            if name not in node._modules:
                node.add_module(name, _Holder())
            node = node._modules[name]
        if kind == "p":
            node.register_parameter(leaf, nn.Parameter(torch.zeros(shape), requires_grad=False))
        elif kind == "b":
            node.register_buffer(leaf, torch.zeros(shape))
        else:
            node.register_buffer(leaf, torch.zeros(shape, dtype=torch.long))


def _conv(p, cout, cin, k):
    return [(p + ".weight", (cout, cin, k), "p"), (p + ".bias", (cout,), "p")]


def _lin(p, cout, cin):
    return [(p + ".weight", (cout, cin), "p"), (p + ".bias", (cout,), "p")]


def _bn(p, c):
    return [(p + ".weight", (c,), "p"), (p + ".bias", (c,), "p"), (p + ".running_mean", (c,), "b"),
            (p + ".running_var", (c,), "b"), (p + ".num_batches_tracked", (), "n")]


def _mlp(p, cin, mid, cout):
    return _lin(p + ".fc1", mid, cin) + _lin(p + ".fc2", cout, mid)


def _mha(p, e):
    return [(p + ".in_proj_weight", (3 * e, e), "p"), (p + ".in_proj_bias", (3 * e,), "p")] + _lin(p + ".out_proj", e, e)


def _tlayer(p, e, ff, cross):
    s = _mha(p + ".self_attn", e)
    if cross:
        s += _mha(p + ".multihead_attn", e)
    s += _lin(p + ".linear1", ff, e) + _lin(p + ".linear2", e, ff)
    for i in range(3 if cross else 2):
        s += [(f"{p}.norm{i + 1}.weight", (e,), "p"), (f"{p}.norm{i + 1}.bias", (e,), "p")]
    return s


def _wav_encoder(p, out_dim):
    chans = [(1, out_dim // 4), (out_dim // 4, out_dim // 4), (out_dim // 4, out_dim // 4),
             (out_dim // 4, out_dim // 2), (out_dim // 2, out_dim // 2), (out_dim // 2, out_dim)]
    s = []
    for i, ((cin, cout), (_, _, has_ds)) in enumerate(zip(chans, E.WAV_BLOCKS)):
        q = f"{p}.feat_extractor.{i}"
        s += _conv(q + ".conv1", cout, cin, 15) + _bn(q + ".bn1", cout)
        s += _conv(q + ".conv2", cout, cout, 15) + _bn(q + ".bn2", cout)
        if has_ds:
            s += _conv(q + ".downsample.0", cout, cin, 15) + _bn(q + ".downsample.1", cout)
    return s


def _resblock(p, c):
    return _conv(p + ".model.0", c, c, 3) + _conv(p + ".model.2", c, c, 3)


def _vq_encoder(p, in_dim, length, n_layer):
    s = []
    for i in range(n_layer):
        s += _conv(f"{p}.main.{3 * i}", length, in_dim if i == 0 else length, 3)
        s += _resblock(f"{p}.main.{3 * i + 2}", length)
    return s


def _vq_decoder(p, out_dim, length, n_layer):
    if n_layer < 1:
        raise ValueError("vae_layer must be >= 1")
    chans = [length] * n_layer + [out_dim]
    s = _resblock(p + ".main.0", length) + _resblock(p + ".main.1", length)
    for i in range(n_layer):
        s += _conv(f"{p}.main.{2 + 2 * i}", chans[i + 1], chans[i], 3)
    s += _conv(f"{p}.main.{2 + 2 * n_layer}", out_dim, out_dim, 3)
    return s


def emage_audio_spec(cfg):
    """Checkpoint layout of EmageAudioModel (M.py:211-263), including the unused template layers
    `transformer_en_layer` / `audio_motion_cross_attn_layer` the reference registers."""
    e, af, mf, cb = cfg.hidden_size, cfg.audio_f, cfg.motion_f, cfg.vae_codebook_size
    ch = cfg.pose_dims + 3 + 4
    s = [("mask_embedding", (1, 1, ch), "p")]
    s += _wav_encoder("audio_encoder_face", af) + _wav_encoder("audio_encoder_body", af)
    s += [("speaker_embedding_body.weight", (cfg.speaker_dims, e), "p"),
          ("speaker_embedding_face.weight", (cfg.speaker_dims, e), "p")]
    s += _vq_encoder("motion_encoder", ch, mf, 3)
    s += _mlp("bodyhints_face", mf, e, mf) + _mlp("bodyhints_body", mf, e, mf)
    s += _lin("audio_body_motion_proj", e, af) + _lin("moton_proj", e, mf)
    s += [("position_embeddings.pe", (1, (cfg.pose_length // cfg.pose_length + 1) * cfg.pose_length, e), "b")]
    s += _tlayer("transformer_en_layer", e, 2 * e, False) + _tlayer("motion_self_encoder.layers.0", e, 2 * e, False)
    s += _tlayer("audio_motion_cross_attn_layer", e, 2 * e, True)
    for i in range(8):
        s += _tlayer(f"audio_motion_cross_attn.layers.{i}", e, 2 * e, True)
    for p in ("upper", "hands", "lower"):
        s += _mlp("motion2latent_" + p, e, e, e)
    for p in ("upper", "hands", "lower"):
        s += _tlayer(f"body_motion_decoder_{p}.layers.0", e, 2 * e, True)
    for p in ("upper", "hands", "lower"):
        s += _lin("motion_out_proj_" + p, cb, e)
    for p in ("upper", "hands", "lower"):
        s += _mlp("motion_cls_" + p, cb, e, cb)
    s += _lin("audio_face_motion_proj", e, af + mf)
    for i in range(4):
        s += _tlayer(f"face_motion_decoder.layers.{i}", e, 2 * e, True)
    s += _lin("face_out_proj", cb, e) + _mlp("face_cls", cb, e, cb)
    return s


def vqvae_spec(cfg, with_quantizer=True):
    s = _vq_encoder("encoder", cfg.vae_test_dim, cfg.vae_length, cfg.vae_layer)
    if with_quantizer:
        s += [("quantizer.embedding.weight", (cfg.vae_codebook_size, cfg.vae_length), "p")]
    return s + _vq_decoder("decoder", cfg.vae_test_dim, cfg.vae_length, cfg.vae_layer)


def _plain_state(module):
    return {k: v.detach() for k, v in module.state_dict().items()}


def _require_cuda(module, what):
    dev = next(module.parameters()).device
    if dev.type != "cuda":
        raise _lib.PmError(f"{what}: module is on {dev}; the GPU path has no CPU fallback - call .to('cuda') first")
    _lib.load()
    return dev


class _EngineOwner(PreTrainedModel):
    """Shared plumbing: build the packed engine lazily, drop it when weights or device change."""

    _engine = None

    def _init_weights(self, module):          # parameters come from checkpoints; nothing to initialise
        pass

    def _invalidate(self):
        self._engine = None

    def load_state_dict(self, *args, **kwargs):
        self._invalidate()
        return super().load_state_dict(*args, **kwargs)

    def _apply(self, fn, *args, **kwargs):
        self._invalidate()
        return super()._apply(fn, *args, **kwargs)


# ----------------------------------------------------------------------------------------------------
# VQ side
# ----------------------------------------------------------------------------------------------------


class EmageVQVAEConv(_EngineOwner):
    """M.py:34-70.  forward()/map2index()/map2latent() (training-side tokenisation, SURVEY section 8f-2)
    use the same kernels; decode()/decode_from_latent() are on the inference path."""
    config_class = EmageVQVAEConvConfig
    base_model_prefix = "emage_vqvaeconv"

    def __init__(self, config):
        super().__init__(config)
        _materialise(self, vqvae_spec(config))
        # attribute surface callers use on the reference's Quantizer (P.py:135-142, M.py:62-64)
        self.quantizer.e_dim = config.vae_length
        self.quantizer.n_e = config.vae_codebook_size
        self.quantizer.beta = config.vae_quantizer_lambda
        self.post_init()

    @property
    def e_dim(self):
        return self.config.vae_length

    def _eng(self):
        if self._engine is None:
            _require_cuda(self, type(self).__name__)
            sd = _plain_state(self)
            self._engine = dict(
                enc=E._ConvStack(sd, "encoder", "encoder", int(self.config.vae_layer)),
                dec=E._ConvStack(sd, "decoder", "decoder", int(self.config.vae_layer)),
                cb=sd["quantizer.embedding.weight"].contiguous(),
            )
            self._engine["e2"] = ops.row_sqnorm(self._engine["cb"])
        return self._engine

    def _index_of(self, latent):
        eng = self._eng()
        if latent.shape[-1] != self.e_dim:
            raise AssertionError("latent last dim must equal e_dim")          # P.py:145,159
        return ops.l2_argmin(latent.contiguous().float(), eng["cb"], eng["e2"])

    def map2index(self, inputs):                                              # M.py:47-50
        eng = self._eng()
        return self._index_of(eng["enc"](inputs.contiguous().float()))

    def map2latent(self, inputs):                                             # M.py:51-55
        eng = self._eng()
        return ops.gather_rows(eng["cb"], self.map2index(inputs))

    def decode(self, index):                                                  # M.py:56-59
        eng = self._eng()
        return eng["dec"](ops.gather_rows(eng["cb"], index.contiguous()))

    def decode_from_latent(self, latent):                                     # M.py:60-70
        return self.decode(self._index_of(latent))

    def forward(self, inputs):                                                # M.py:42-46
        eng = self._eng()
        pre = eng["enc"](inputs.contiguous().float())
        index = self._index_of(pre)
        z_q = ops.gather_rows(eng["cb"], index)
        # loss / perplexity / the straight-through value are training-side bookkeeping off the inference path
        # (P.py:151-155): plain torch.  The decoder sees z + (z_q - z), as in the reference, not the bare code.
        beta = float(self.config.vae_quantizer_lambda)
        loss = torch.mean((z_q - pre) ** 2) + beta * torch.mean((z_q - pre) ** 2)
        z_st = (pre + (z_q - pre)).contiguous()
        e_mean = torch.bincount(index.reshape(-1), minlength=eng["cb"].shape[0]).float() / index.numel()
        perplexity = torch.exp(-torch.sum(e_mean * torch.log(e_mean + 1e-10)))
        return {"poses_feat": z_st, "embedding_loss": loss, "perplexity": perplexity, "rec_pose": eng["dec"](z_st)}


class EmageVAEConv(_EngineOwner):
    """M.py:19-32."""
    config_class = EmageVAEConvConfig
    base_model_prefix = "emage_vaeconv"

    def __init__(self, config):
        super().__init__(config)
        _materialise(self, vqvae_spec(config, with_quantizer=False))
        self.post_init()

    def _eng(self):
        if self._engine is None:
            _require_cuda(self, type(self).__name__)
            sd = _plain_state(self)
            n = int(self.config.vae_layer)
            self._engine = (E._ConvStack(sd, "encoder", "encoder", n), E._ConvStack(sd, "decoder", "decoder", n))
        return self._engine

    def forward(self, inputs):
        enc, dec = self._eng()
        return {"rec_pose": dec(enc(inputs.contiguous().float()))}


class EmageVQModel(nn.Module):
    """M.py:72-205: the four body-part VQ-VAEs + the global-motion auto-encoder."""

    def __init__(self, face_model, upper_model, hands_model, lower_model, global_model):
        super().__init__()
        self.joint_mask_upper = [j in (3, 6, 9, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21) for j in range(55)]
        self.joint_mask_lower = [j in (0, 1, 2, 4, 5, 7, 8, 10, 11) for j in range(55)]
        self.vq_model_face = face_model
        self.vq_model_upper = upper_model
        self.vq_model_hands = hands_model
        self.vq_model_lower = lower_model
        self.global_motion = global_model
        self._engine = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._engine = None
        return super().load_state_dict(*a, **k)

    def engine(self) -> E.VQEngine:
        if self._engine is None:
            parts = dict(face=self.vq_model_face, upper=self.vq_model_upper, hands=self.vq_model_hands,
                         lower=self.vq_model_lower)
            for m in parts.values():
                _require_cuda(m, "EmageVQModel")
            sds = {p: _plain_state(m) for p, m in parts.items()}
            cfgs = {p: m.config.to_dict() for p, m in parts.items()}
            if self.global_motion is not None:
                sds["global"] = _plain_state(self.global_motion)
                cfgs["global"] = self.global_motion.config.to_dict()
            self._engine = E.VQEngine(sds, cfgs)
        return self._engine

    # -- training-side tokenisation (M.py:97-124); not on the inference path ---------------------------
    def spilt_inputs(self, smplx_body_rot6d, expression, tar_contact=None, tar_trans=None):
        bs, t, j6 = smplx_body_rot6d.shape
        r = smplx_body_rot6d.reshape(bs, t, j6 // 6, 6)
        dev = r.device
        upper_j = [j for j, m in enumerate(self.joint_mask_upper) if m]
        lower_j = [j for j, m in enumerate(self.joint_mask_lower) if m]
        tar_contact = torch.zeros(bs, t, 4, device=dev) if tar_contact is None else tar_contact
        tar_trans = torch.zeros(bs, t, 3, device=dev) if tar_trans is None else tar_trans
        return dict(face=torch.cat([r[:, :, 22].reshape(bs, t, 6), expression], dim=2),
                    upper=r[:, :, upper_j].reshape(bs, t, 78), hands=r[:, :, 25:55].reshape(bs, t, 180),
                    lower=torch.cat([r[:, :, lower_j].reshape(bs, t, 54), tar_trans, tar_contact], dim=2))

    def map2index(self, smplx_body_rot6d, expression, tar_contact=None, tar_trans=None):
        x = self.spilt_inputs(smplx_body_rot6d, expression, tar_contact, tar_trans)
        return dict(face=self.vq_model_face.map2index(x["face"]), upper=self.vq_model_upper.map2index(x["upper"]),
                    hands=self.vq_model_hands.map2index(x["hands"]), lower=self.vq_model_lower.map2index(x["lower"]))

    def map2latent(self, smplx_body_rot6d, expression, tar_contact=None, tar_trans=None):
        x = self.spilt_inputs(smplx_body_rot6d, expression, tar_contact, tar_trans)
        return dict(face=self.vq_model_face.map2latent(x["face"]), upper=self.vq_model_upper.map2latent(x["upper"]),
                    hands=self.vq_model_hands.map2latent(x["hands"]), lower=self.vq_model_lower.map2latent(x["lower"]))

    # -- inference path ---------------------------------------------------------------------------------
    def decode(self, face_index=None, upper_index=None, hands_index=None, lower_index=None,
               face_latent=None, upper_latent=None, hands_latent=None, lower_latent=None,
               get_global_motion=False, ref_trans=None):
        """M.py:126-193: index (preferred) or latent per part -> expression, all_motion4inference,
        motion_axis_angle, trans."""
        index = dict(face=face_index, upper=upper_index, hands=hands_index, lower=lower_index)
        latent = dict(face=face_latent, upper=upper_latent, hands=hands_latent, lower=lower_latent)
        if all(v is None for v in list(index.values()) + list(latent.values())):
            raise UnboundLocalError("decode() needs at least one index or latent (bs, t undefined)")   # M.py:130-133
        for p in index:                      # an index takes precedence over a latent (M.py:135-139)
            if index[p] is not None:
                latent[p] = None
        return self.engine().decode(index, latent, get_global_motion=get_global_motion, ref_trans=ref_trans)

    def get_global_motion(self, lower_body, ref_trans):
        return self.engine().global_motion(lower_body.contiguous().float(), ref_trans)


# ----------------------------------------------------------------------------------------------------
# The audio -> token model
# ----------------------------------------------------------------------------------------------------


class EmageAudioModel(_EngineOwner):
    """M.py:208-490."""
    config_class = EmageAudioConfig
    base_model_prefix = "emage_audio"

    def __init__(self, config: EmageAudioConfig):
        super().__init__(config)
        self.cfg = config
        _materialise(self, emage_audio_spec(config))
        from .pe import periodic_table
        period = config.pose_length
        self.position_embeddings.pe.copy_(periodic_table(config.hidden_size, period).repeat(
            self.position_embeddings.pe.shape[1] // period, 1).unsqueeze(0))
        self.post_init()

    def _eng(self) -> E.EmageEngine:
        if self._engine is None:
            _require_cuda(self, "EmageAudioModel")
            self._engine = E.EmageEngine(_plain_state(self), self.cfg.to_dict())
        return self._engine

    def forward(self, audio, speaker_id, masked_motion, mask, use_audio=True):
        """One window (M.py:265-341): audio (bs, n), speaker_id (bs,1) long, masked_motion / mask (bs,T,337)
        with mask==1 meaning "masked".  Returns the 8 rec_*/cls_* tensors (bs,T,256)."""
        eng = self._eng()
        dev = eng.device
        audio = audio.to(device=dev, dtype=torch.float32).contiguous()
        motion = masked_motion.to(device=dev, dtype=torch.float32).contiguous()
        mask = mask.to(device=dev, dtype=torch.float32).contiguous()
        bs, t, ch = motion.shape
        # no seed splice here: pre = 0 makes window_input the plain `where(mask==1, embedding, motion)`

        def run():
            win_in = ops.window_input(motion, mask, None, eng.mask_embedding, 0, t, 0, nsplit=E._ns(), f32=False)
            mem_face, kv = eng.audio_phase(audio, 0, 0, 1, audio.shape[1], t)
            return eng.window(win_in, eng.speaker_rows(speaker_id.to(dev)), mem_face, kv, use_audio=use_audio)
        return E.guarded(run, lambda out: [out["cls_" + p] for p in E.PARTS])

    def inference(self, audio, speaker_id, vq_model, masked_motion=None, mask=None):
        """Sliding-window generation (M.py:343-490)."""
        return E.guarded(lambda: E.run_inference(self._eng(), vq_model.engine(), audio, speaker_id, masked_motion, mask),
                         lambda out: [out["cls_" + p] for p in E.PARTS])
