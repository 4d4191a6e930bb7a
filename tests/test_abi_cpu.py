"""CPU-only checks: the C-ABI library builds (nvcc cross-compile), loads and exports every symbol
include/zeggs_b200.h declares; host-side table construction matches the oracle; no compute calls."""
import json
import os
import re

import numpy as np
import pytest

from tests._util import ROOT, ensure_built


@pytest.fixture(scope="module")
def built():
    ensure_built()
    from zeggs_b200 import _lib
    return _lib


def test_library_exports_every_header_symbol(built):
    hdr = open(os.path.join(ROOT, "include", "zeggs_b200.h")).read()
    declared = set(re.findall(r"\b(zeggs_[a-z0-9_]+)\s*\(", hdr))
    l = built.lib()
    bound = {s[0] for s in built.SYMBOLS}
    assert declared == bound, (declared - bound, bound - declared)
    for name in declared:
        assert getattr(l, name) is not None
    assert l.zeggs_version() >= 100


def test_ctypes_mirrors_have_the_library_struct_layout(built):
    """Every args struct of the header is mirrored in _lib.py: same size as the compiled C struct (a drifted mirror would make the
    library read garbage pointers), and every struct the header defines has a mirror."""
    import ctypes
    hdr = open(os.path.join(ROOT, "include", "zeggs_b200.h")).read()
    defined = set(re.findall(r"^\}\s*(zeggs_[a-z0-9_]+);", hdr, flags=re.M))
    mirrors = built.struct_mirrors()
    assert defined == set(mirrors), (defined - set(mirrors), set(mirrors) - defined)
    l = built.lib()
    for name, cls in mirrors.items():
        assert l.zeggs_struct_size(name.encode()) == ctypes.sizeof(cls), name
    assert l.zeggs_struct_size(b"no_such_struct") == 0


def test_mel_frame_count_rule(built):
    l = built.lib()
    from oracle import mel_oracle
    for ns, hop in [(160000, 200), (160000, 160), (16001, 200), (12345, 160), (800, 200), (500, 200)]:
        assert l.zeggs_mel_num_frames(ns, 800, hop) == mel_oracle.num_frames(ns, 800, hop)


def _size_table(l):
    """Every *_bytes query of the header over a small grid of shapes (zeros included), keyed by query name: the layouts of the
    workspaces and packed weights are part of the ABI, and phase 2 of the decoder backward relies on the same carve-up as phase 1."""
    Hs, Bs, Ts, Zs, S = (16, 64, 384, 1024, 1056, 1072, 2112, 2128), (1, 32, 33), (1, 2, 256), (9, 64), 64
    q = lambda name, shapes: [int(getattr(l, "zeggs_" + name)(*s)) for s in shapes]
    packed = [(H, S, Z) for H in Hs for Z in Zs]
    ws = [(B, T, H, S, Z) for H in Hs for B in Bs for T in Ts for Z in Zs]
    ws_save = [s + (save,) for s in ws for save in (0, 1)]
    t = {name: q(name, packed) for name in ("decoder_packed_bytes", "decoder_packed_tc_bytes", "decoder_tc_workspace_bytes",
                                            "decoder_packed_bwd_bytes", "decoder_packed_bwd_tc_bytes", "decoder_bwd_tc_workspace_bytes",
                                            "decoder_packed_film_bytes", "decoder_packed_bwd_film_bytes")}
    t.update({name: q(name, ws_save) for name in ("decoder_workspace_bytes", "decoder_film_workspace_bytes")})
    t.update({name: q(name, ws) for name in ("decoder_bwd_workspace_bytes", "decoder_film_bwd_workspace_bytes")})
    t["speech_enc_workspace_bytes"] = q("speech_enc_workspace_bytes", [(1, 1, 80, 64, 64), (32, 34, 81, 128, 64), (64, 256, 80, 256, 128),
                                                                       (0, 34, 81, 128, 64)])
    t["style_enc_workspace_bytes"] = q("style_enc_workspace_bytes", [(1, 1, 1134, 256, 128, 2), (32, 256, 1134, 256, 128, 2),
                                                                     (7, 33, 1131, 64, 64, 4), (7, 33, 1131, 64, 63, 4)])
    t["style_enc_gru_workspace_bytes"] = q("style_enc_gru_workspace_bytes", [(1, 1, 1134, 64, 64, 0), (32, 256, 1134, 1056, 128, 1),
                                                                             (1216, 17, 1134, 1056, 128, 1), (33, 2, 10, 528, 9, 0),
                                                                             (33, 2, 10, 528, 9, 1), (1, 1, 1134, 532, 64, 0)])
    t["loss_workspace_bytes"] = q("loss_workspace_bytes", [(1, 1), (32, 256), (33, 2), (0, 5)])
    t["loudness_workspace_bytes"] = q("loudness_workspace_bytes", [(1, 1), (4, 100), (32, 1000), (0, 10)])
    t["anim_features_workspace_bytes"] = q("anim_features_workspace_bytes", [(1, 75), (256, 75), (1000, 3), (0, 75)])
    t["spline_resample_workspace_bytes"] = q("spline_resample_workspace_bytes", [(1, 1), (1000, 1131), (10 ** 6, 3), (0, 3)])
    t["masked_moments_workspace_bytes"] = q("masked_moments_workspace_bytes", [(1, 1), (1000, 1131), (10 ** 6, 75), (0, 75)])
    return t


def test_workspace_and_pack_sizes_match_golden(built):
    l = built.lib()
    assert l.zeggs_decoder_packed_bytes(1024, 64, 64) > 4 * (1024 * 1134 * 4 + 12 * 1024 * 1024)
    assert l.zeggs_decoder_packed_bytes(1000, 64, 64) == 0          # H % 16 != 0 -> unsupported
    a = l.zeggs_decoder_workspace_bytes(32, 256, 1024, 64, 64, 1)
    b = l.zeggs_decoder_workspace_bytes(32, 256, 1024, 64, 64, 0)
    assert a > b > 0
    # the exact sizes: any change to a workspace or pack layout shows up here
    with open(os.path.join(ROOT, "tests", "golden", "workspace_sizes.json")) as f:
        want = json.load(f)
    got = _size_table(l)
    hdr = open(os.path.join(ROOT, "include", "zeggs_b200.h")).read()
    assert set(got) == {n[len("zeggs_"):] for n in re.findall(r"\b(zeggs_[a-z0-9_]+_bytes)\s*\(", hdr)}
    assert got == want


def test_style_gru_refuses_batches_its_backward_cannot_hold(built):
    """The GRU encoder's BPTT kernel keeps a carry of U*32 floats per 32-sample tile in shared memory, so at H = 1056 (U = 8) one call
    takes at most 1216 samples on an H100 (227 KB per block).  The workspace query reports 0 and both entry points refuse a larger
    batch, naming the limit, before they launch anything (before, the backward failed at cudaFuncSetAttribute after the forward ran)."""
    import ctypes
    l = built.lib()
    assert l.zeggs_style_enc_gru_workspace_bytes(1216, 17, 1134, 1056, 128, 1) > 0
    assert l.zeggs_style_enc_gru_workspace_bytes(1217, 17, 1134, 1056, 128, 1) == 0
    assert l.zeggs_style_enc_gru_workspace_bytes(7936, 17, 1134, 528, 128, 1) > 0        # U = 4: 248 tiles
    assert l.zeggs_style_enc_gru_workspace_bytes(7937, 17, 1134, 528, 128, 1) == 0
    assert l.zeggs_style_enc_gru_workspace_bytes(1, 17, 1134, 532, 128, 1) == 0          # unsupported hidden size
    dummy = ctypes.create_string_buffer(64)
    p = ctypes.addressof(dummy)
    a = built.StyleEncGruArgs(B=1217, T=17, C_in=1134, H=1056, E=128, temperature=1.0, x=p, z=p, mu=p, logvar=p, workspace=p,
                              workspace_bytes=1 << 40)
    g = built.StyleEncGruGrads(dz=p, dmu=p, dlogvar=p)
    launches = l.zeggs_launch_count()
    assert l.zeggs_style_enc_gru_fwd(ctypes.byref(a), None) != 0
    assert "at most 1216 samples" in l.zeggs_last_error().decode()
    assert l.zeggs_style_enc_gru_bwd(ctypes.byref(a), ctypes.byref(g), None) != 0
    assert "at most 1216 samples" in l.zeggs_last_error().decode()
    assert l.zeggs_launch_count() == launches


def test_host_filterbank_matches_oracle():
    from oracle import mel_oracle
    from zeggs_b200.audio import mel_filterbank
    a = mel_filterbank(800, 16000, 80, 20, 7600, True)
    b = mel_oracle.mel_filterbank(800, 16000, 80, 20, 7600, True)
    assert np.array_equal(a, b)
    assert int((a != 0).sum()) == 742          # SURVEY.md 8a (a2)


def test_compute_path_refuses_cpu_tensors(built):
    import torch
    from zeggs_b200 import modules, _lib
    dec = modules.Decoder(1134, 1131, 64, 64, 64, 2)
    z = torch.zeros
    with pytest.raises(_lib.ZeggsError):
        dec(z(1, 3), z(1, 4), z(1, 3), z(1, 3), z(1, 75, 3), z(1, 75, 2, 3), z(1, 75, 3), z(1, 75, 3), z(1, 4, 3),
            z(1, 4, 64), z(1, 4, 64), None, z(1134), torch.ones(1134), z(1131), torch.ones(1131), 1 / 60)
