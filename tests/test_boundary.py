"""Drop-in boundary checks that need no GPU: checkpoint layout, export list, C-ABI symbols,
loud failure without CUDA."""
import ctypes
import json
import os
import re

import pytest
import torch

from oracle.weights import EMAGE_CFG, VQ_CFGS, load_manifest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _models():
    from pantomatrix_b200.emage_audio import (EmageAudioConfig, EmageAudioModel, EmageVAEConv, EmageVAEConvConfig,
                                              EmageVQVAEConv, EmageVQVAEConvConfig)
    out = {"emage": EmageAudioModel(EmageAudioConfig(**EMAGE_CFG))}
    for p in ("face", "upper", "hands", "lower"):
        out["vq_" + p] = EmageVQVAEConv(EmageVQVAEConvConfig(**VQ_CFGS[p]))
    out["vq_global"] = EmageVAEConv(EmageVAEConvConfig(**VQ_CFGS["global"]))
    from oracle.weights import LSTM_CFG
    from pantomatrix_b200.lstm_audio import CamnAudioConfig, CamnAudioModel, DiscoAudioConfig, DiscoAudioModel
    out["camn"] = CamnAudioModel(CamnAudioConfig(**LSTM_CFG))
    out["disco"] = DiscoAudioModel(DiscoAudioConfig(**LSTM_CFG))
    return out


def test_state_dict_layout_matches_reference():
    """Keys, shapes and dtypes equal the reference checkpoints (manifest recorded from the live reference
    modules), so reference checkpoints load with strict=True."""
    man = load_manifest()
    for tag, module in _models().items():
        sd = module.state_dict()
        want = {k: tuple(s) for k, s in man[tag]}
        assert set(sd) == set(want), (tag, sorted(set(sd) ^ set(want))[:10])
        for k, v in sd.items():
            assert tuple(v.shape) == want[k], (tag, k, v.shape, want[k])
            assert v.dtype == (torch.int64 if k.endswith("num_batches_tracked") else torch.float32)


def test_positional_table_is_bit_identical_to_oracle():
    from oracle.emage_oracle import pos_table
    from pantomatrix_b200.emage_audio.pe import periodic_table
    assert torch.equal(periodic_table(768, 64), pos_table(768, 64))


def test_export_list_and_shim():
    import models.emage_audio as shim
    import pantomatrix_b200.emage_audio as pkg
    names = ["EmageAudioConfig", "EmageAudioModel", "EmageVQVAEConvConfig", "EmageVQVAEConv", "EmageVQModel",
             "EmageVAEConvConfig", "EmageVAEConv"]
    assert sorted(pkg.__all__) == sorted(names)
    for n in names:
        assert getattr(shim, n) is getattr(pkg, n)
    import models.camn_audio as camn
    import models.disco_audio as disco
    assert sorted(camn.__all__) == ["CamnAudioConfig", "CamnAudioModel", "CamnAudioPreTrainedModel"]
    assert sorted(disco.__all__) == ["DiscoAudioConfig", "DiscoAudioModel", "DiscoAudioPreTrainedModel"]


def test_save_and_from_pretrained_round_trip(tmp_path):
    from pantomatrix_b200.emage_audio import EmageVQVAEConv, EmageVQVAEConvConfig
    from oracle.weights import load_synthetic
    m = load_synthetic(EmageVQVAEConv(EmageVQVAEConvConfig(**VQ_CFGS["face"])), 3, "vq_face")
    m.save_pretrained(tmp_path / "emage_vq" / "face")
    assert sorted(os.listdir(tmp_path / "emage_vq" / "face")) == ["config.json", "model.safetensors"]
    m2 = EmageVQVAEConv.from_pretrained(str(tmp_path), subfolder="emage_vq/face")     # T.py:82 call form
    for (k, a), (_, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert torch.equal(a, b), k
    assert m2.quantizer.e_dim == 256 and m2.quantizer.embedding.weight.shape == (256, 256)


def test_library_exports_every_declared_symbol_at_the_header_abi_version():
    """Every function declared in include/pm_emage.h is exported by the built library and bound in
    pantomatrix_b200._lib, and the library reports the header's ABI version, 6 (no compute call is made: there is no
    GPU here)."""
    from pantomatrix_b200 import _lib, build
    build.build()
    header = open(os.path.join(ROOT, "include", "pm_emage.h")).read()
    declared = set(re.findall(r"^int\s+(pm_\w+)\s*\(", header, flags=re.M))
    assert declared, "no declarations found"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in pm_emage.h but not exported"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert re.search(r"^#define PM_ABI_VERSION (\d+)$", header, flags=re.M).group(1) == "6"
    assert _lib.load().pm_abi_version() == 6


def test_ctypes_signatures_match_the_header():
    """Argument-by-argument: the ctypes binding of every entry point has the C types of its declaration in
    include/pm_emage.h, and the definitions in csrc/ repeat the declaration (a drifted float / int here would
    corrupt every later argument of a call)."""
    import glob
    from pantomatrix_b200 import _lib

    def protos(text):
        out = {}
        for name, args in re.findall(r"\bint\s+(pm_\w+)\s*\(([^)]*)\)", re.sub(r"/\*.*?\*/", "", text, flags=re.S)):
            kinds = []
            for a in (x.strip() for x in args.split(",")):
                if a in ("void", ""):
                    continue
                kinds.append("p" if "*" in a else "ll" if "long long" in a else "f" if a.startswith("float") else "i")
            out[name] = kinds
        return out

    tag = {ctypes.c_void_p: "p", ctypes.c_longlong: "ll", ctypes.c_float: "f", ctypes.c_int: "i"}
    header = protos(open(os.path.join(ROOT, "include", "pm_emage.h")).read())
    for name, args in _lib.SIGNATURES.items():
        assert [tag[a] for a in args] == header[name], name
    defined = {}
    for f in glob.glob(os.path.join(ROOT, "pantomatrix_b200", "csrc", "*.cu")):
        src = open(f).read()
        src = re.sub(r"//[^\n]*", "", src)
        defined.update(protos(src.replace('extern "C" int', "int")))
    for name, kinds in header.items():
        assert defined.get(name) == kinds, (name, defined.get(name), kinds)


def test_ops_call_sites_pass_the_declared_number_of_arguments():
    """Every `_call("pm_...", ...)` in pantomatrix_b200/ops.py passes as many arguments as the binding declares
    (`*_pargs(...)` expands to the 4 plane arguments) - checked statically, since no kernel can be launched here."""
    import ast
    from pantomatrix_b200 import _lib
    tree = ast.parse(open(os.path.join(ROOT, "pantomatrix_b200", "ops.py")).read())
    seen = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and getattr(node.func, "id", None) == "_call":
            name = node.args[0].value
            n = sum(4 if isinstance(a, ast.Starred) else 1 for a in node.args[1:])
            assert n == len(_lib.SIGNATURES[name]), (name, n, len(_lib.SIGNATURES[name]))
            seen.add(name)
    # pm_memset_async is not a kernel launch: ops.py reaches it through _lib.call, not through the counting _call
    assert seen == set(_lib.SIGNATURES) - {"pm_abi_version", "pm_device_cc", "pm_memset_async"}, seen ^ set(_lib.SIGNATURES)


def test_ops_wrappers_marshal_valid_arguments(monkeypatch):
    """The real pantomatrix_b200.ops wrappers (not the fake ones) executed on CPU tensors with the library call
    replaced by a recorder: every argument must convert to the ctypes type its binding declares, for bf16 and fp16
    planes.  Catches marshalling mistakes (a tensor where a pointer is due, None for an int, a missing argument)
    without a GPU; the kernels themselves are covered by the -m gpu tests."""
    from pantomatrix_b200 import _lib, ops
    calls = []

    def record(name, *args):
        sig = _lib.SIGNATURES[name]
        assert len(args) == len(sig), (name, len(args), len(sig))
        for i, (a, t) in enumerate(zip(args, sig)):
            if t is ctypes.c_void_p:
                assert a is None or isinstance(a, int), (name, i, type(a))
            elif t is ctypes.c_float:
                assert isinstance(a, float), (name, i, type(a))
            else:
                assert isinstance(a, int) and not isinstance(a, bool), (name, i, type(a))
                t(a)
        calls.append((name, args))

    monkeypatch.setattr(_lib, "call", record)
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=torch.float32: t)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_PLANE_DTYPE", ops._PLANE_DTYPE)
    for fmt, bit in (("bf16", 0), ("fp16", ops.FMT_F16)):
        ops.set_plane_format(fmt)
        calls.clear()
        x = torch.zeros(2, 64, 768)
        pl = ops.split_bf16(x, 2)
        w = ops.PackedW(torch.randn(1, 768, 768) * 0.03, 2)
        assert (w.acc_scale == 1.0) == (fmt == "bf16")
        out, planes = ops.tapgemm_tc(pl, w, torch.zeros(768), rows_out=64, act=ops.ACT_RELU, residual=torch.zeros(2, 64, 768),
                                     out_nsplit=2)
        assert out.shape == (2, 64, 768) and planes.t.dtype == pl.t.dtype
        ln = ops.add_layernorm(x, x, torch.ones(768), torch.zeros(768), nsplit=2)
        att = ops.attention(x.view(128, 768), x.view(128, 768), x.view(128, 768), 2, 4, 64, 64, 192, nsplit=2, f32=False)
        ops.add2(x, x, nsplit=2)
        ops.gather_rows(torch.zeros(256, 256), torch.zeros(2, 8, dtype=torch.long), nsplit=2)
        assert ln.p.t.dtype == att.p.t.dtype == pl.t.dtype
        by_name = dict(calls)
        assert by_name["pm_split_bf16"][10] == 2 | bit
        gemm = by_name["pm_tapgemm_tc"]
        assert gemm[13] == 2 | bit and gemm[31] == 2 | bit and gemm[23] == float(w.acc_scale)
        assert by_name["pm_add_layernorm_f32"][11] == 2 | bit and by_name["pm_attention_f32"][16] == 2 | bit


def test_no_cpu_fallback():
    """The product path must fail loudly off-GPU instead of computing on the CPU."""
    from pantomatrix_b200 import _lib
    m = _models()
    vq = m["vq_face"]
    with pytest.raises(_lib.PmError):
        vq.decode(torch.zeros(1, 8, dtype=torch.long))
    with pytest.raises(_lib.PmError):
        m["emage"].forward(torch.zeros(1, 34112), torch.zeros(1, 1, dtype=torch.long),
                           torch.zeros(1, 64, 337), torch.ones(1, 64, 337))


def test_product_never_imports_the_oracle():
    for base, _, files in os.walk(os.path.join(ROOT, "pantomatrix_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(base, f)).read()
                assert "oracle" not in src.replace("no oracle", ""), os.path.join(base, f)
