"""The C-ABI shared library loads without a GPU and exports every symbol include/must3r_b200.h declares
(no compute calls here), the ctypes structs have the C layout, and the product path refuses to run on CPU."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "must3r_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(m3r_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_at_abi_5_and_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    from must3r_b200 import _lib
    import must3r_b200.model  # noqa: F401
    lib = _lib.lib()
    names = declared_functions()
    assert len(names) >= 16
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature"
    assert lib.m3r_abi_version() == 5


def test_ctypes_structs_match_the_c_layout(tmp_path):
    """Compile a tiny C program against the header and compare sizeof() of every struct with ctypes."""
    from must3r_b200 import _lib
    from must3r_b200.model import common as cm
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "must3r_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n",'
                    'sizeof(m3r_gemm_group),sizeof(m3r_gemm_args),sizeof(m3r_attn_args),sizeof(m3r_enc_block),sizeof(m3r_encoder_weights),'
                    'sizeof(m3r_dec_block),sizeof(m3r_decoder_weights),sizeof(m3r_dec_group),sizeof(m3r_decoder_call));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    got = [C.sizeof(t) for t in (_lib.GemmGroup, _lib.GemmArgs, _lib.AttnArgs, cm.EncBlock, cm.EncoderWeights, cm.DecBlock,
                                 cm.DecoderWeights, cm.DecGroup, cm.DecoderCall)]
    assert got == sizes


def test_product_path_fails_loudly_without_cuda():
    from must3r_b200 import ops, synthetic as syn
    from must3r_b200.model import Dust3rEncoder, MUSt3R
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.layernorm(torch.zeros(4, 64), torch.ones(64), torch.zeros(64), 1e-6)
    enc = Dust3rEncoder(img_size=(64, 64), embed_dim=128, depth=1, num_heads=2)
    imgs, ts = syn.synthetic_views(1, 32, 48)
    with pytest.raises(RuntimeError, match="CUDA only"):
        enc(imgs, ts)
    dec = MUSt3R(img_size=(64, 64), enc_embed_dim=128, embed_dim=128, depth=1, num_heads=2, memory_mode="kv", landscape_only=False)
    with pytest.raises(RuntimeError, match="CUDA only"):
        dec(torch.zeros(1, 1, 6, 128), torch.zeros(1, 1, 6, 2, dtype=torch.int64), ts[None], None)


def test_load_model_arg_rewrites():
    """convert_decoder_args / set_image_size_in_args behave like must3r/model/__init__.py:53-108."""
    from must3r_b200.model import convert_decoder_args, set_image_size_in_args
    d = convert_decoder_args("CausalMUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode=\"kv\")")
    assert d.startswith("MUSt3R(") and d.endswith(",landscape_only=False)")
    e = set_image_size_in_args("Dust3rEncoder(img_size=(512, 512), pos_embed='RoPE100')", 768, verbose=False)
    assert "img_size=(768,768)" in e and "pos_embed='RoPE100_512:768'" in e
    e = set_image_size_in_args("Dust3rEncoder(img_size=(224, 224))", 512, verbose=False)
    assert e.endswith(",pos_embed='RoPE100_224:512')")
    with pytest.raises(ValueError):
        set_image_size_in_args("Dust3rEncoder()", 512, verbose=False)


def test_state_dict_keys_are_the_references():
    """Key names/shapes of SURVEY.md §3.1 (292 encoder tensors, 301 decoder tensors)."""
    from must3r_b200.model import Dust3rEncoder, MUSt3R
    from must3r_b200 import synthetic as syn
    enc = Dust3rEncoder()
    dec = MUSt3R(feedback_type="single_mlp", memory_mode="kv")
    assert len(enc.state_dict()) == 292 and len(dec.state_dict()) == 301
    enc.load_state_dict(syn.encoder_state_dict(0), strict=True)
    dec.load_state_dict(syn.decoder_state_dict(0), strict=True)
    assert float(dec.feedback_layer.fc2.weight.abs().sum()) > 0
    fresh = MUSt3R(feedback_type="single_mlp")
    assert float(fresh.feedback_layer.fc2.weight.abs().sum()) == 0      # feedback_mechanism.py:26-35


def test_constructor_string_rewrites_match_reference():
    """set_image_size_in_args / convert_decoder_args (must3r/model/__init__.py:53-108) against strings produced by the
    reference's own functions (tests/golden/model_args.json, generated in the build container)."""
    import json
    from must3r_b200.model import set_image_size_in_args, convert_decoder_args, get_dtype
    g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "model_args.json")))
    for args, size, want in g["set_image_size"]:
        assert set_image_size_in_args(args, size, verbose=False) == want, (args, size)
    for args, want in g["convert"]:
        assert convert_decoder_args(args) == want, args
    with pytest.raises(ValueError):
        set_image_size_in_args("MUSt3R()", 224, verbose=False)
    assert get_dtype("fp16") == torch.float16 and get_dtype("bf16") == torch.bfloat16 and get_dtype(None) == torch.float32

