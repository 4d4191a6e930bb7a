"""Seeded synthetic weights and inputs of the reference's shapes (SURVEY.md §8d).

numpy-only (no torch RNG) so the same bytes are produced in the dev container and on
the GPU box.  Keys of the parameter dict are the reference state-dict names (SURVEY.md
§8b) prefixed with "speech_encoder." / "style_encoder." / "decoder.".
"""
import os

import numpy as np

NJ = 75
P_IN = 6 + NJ * 15 + 3      # 1134  (modules.py:699-710)
P_OUT = 6 + NJ * 15         # 1131  (modules.py:731-736)
N_AUDIO = 81

_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "pose_stats_v1.npz")


def load_stats():
    """Normalisation vectors + skeleton of the shipped processed_v1 (stats.npz, data_definition.json)."""
    s = np.load(_DATA)
    return {k: s[k] for k in s.files}


def _u(rs, shape, bound):
    return rs.uniform(-bound, bound, size=shape).astype(np.float32)


def make_params(H=1024, S=64, Z=64, style_hidden=512, style_embed=128, seed=1234, with_style=True, style_type="attn",
                rnn_cond="normal"):
    """Random weights with PyTorch-default-like scales for every tensor on the path.  style_embed is the style encoder's
    output size (2*Z with the VAE, Z without); style_type 'attn' (StyleEncoderAttn) or 'gru' (StyleEncoderGRU); rnn_cond
    'normal' (RecurrentDecoderNormal) or 'film' (RecurrentDecoderFiLM: its tensors come from a generator of their own, every other
    tensor is the one rnn_cond='normal' gives)."""
    rs = np.random.RandomState(seed)
    A = P_IN + S + Z
    P = {}
    # SpeechEncoder (modules.py:250-263)
    P["speech_encoder.layer0.weight"] = _u(rs, (S, N_AUDIO, 1), 1 / np.sqrt(N_AUDIO))
    P["speech_encoder.layer0.bias"] = _u(rs, (S,), 1 / np.sqrt(N_AUDIO))
    P["speech_encoder.layer1.weight"] = _u(rs, (S, S, 31), 1 / np.sqrt(S * 31))
    P["speech_encoder.layer1.bias"] = _u(rs, (S,), 1 / np.sqrt(S * 31))
    P["speech_encoder.layer2.weight"] = _u(rs, (S, S), 1 / np.sqrt(S))
    P["speech_encoder.layer2.bias"] = _u(rs, (S,), 1 / np.sqrt(S))
    # Decoder (modules.py:165-185, 230-243)
    d = "decoder.recurrent_decoder."
    P[d + "layer0.weight"] = _u(rs, (H, A), 1 / np.sqrt(A))
    P[d + "layer0.bias"] = _u(rs, (H,), 1 / np.sqrt(A))
    kb = 1 / np.sqrt(H)
    P[d + "layer1.weight_ih_l0"] = _u(rs, (3 * H, A + H), kb)
    P[d + "layer1.weight_hh_l0"] = _u(rs, (3 * H, H), kb)
    P[d + "layer1.bias_ih_l0"] = _u(rs, (3 * H,), kb)
    P[d + "layer1.bias_hh_l0"] = _u(rs, (3 * H,), kb)
    P[d + "layer1.weight_ih_l1"] = _u(rs, (3 * H, H), kb)
    P[d + "layer1.weight_hh_l1"] = _u(rs, (3 * H, H), kb)
    P[d + "layer1.bias_ih_l1"] = _u(rs, (3 * H,), kb)
    P[d + "layer1.bias_hh_l1"] = _u(rs, (3 * H,), kb)
    P[d + "layer2.weight"] = _u(rs, (P_OUT, H), kb)
    P[d + "layer2.bias"] = _u(rs, (P_OUT,), kb)
    c = "decoder.cell_state_encoder."
    P[c + "layer0.weight"] = _u(rs, (H, P_IN + Z), 1 / np.sqrt(P_IN + Z))
    P[c + "layer0.bias"] = _u(rs, (H,), 1 / np.sqrt(P_IN + Z))
    P[c + "layer1.weight"] = _u(rs, (H, H), kb)
    P[c + "layer1.bias"] = _u(rs, (H,), kb)
    P[c + "layer2.weight"] = _u(rs, (2 * H, H), kb)
    P[c + "layer2.bias"] = _u(rs, (2 * H,), kb)
    if with_style and style_type == "gru":
        E, Hs = style_embed, style_hidden
        e = "style_encoder.encoder."
        xav = lambda co, ci, k, gain: gain * np.sqrt(6.0 / (ci * k + co * k))
        P[e + "convs.0.conv.weight"] = _u(rs, (Hs, P_IN, 3), xav(Hs, P_IN, 3, np.sqrt(2)))
        P[e + "convs.0.conv.bias"] = _u(rs, (Hs,), 1 / np.sqrt(P_IN * 3))
        P[e + "convs.2.conv.weight"] = _u(rs, (Hs, Hs, 3), xav(Hs, Hs, 3, np.sqrt(2)))
        P[e + "convs.2.conv.bias"] = _u(rs, (Hs,), 1 / np.sqrt(Hs * 3))
        for sfx in ("", "_reverse"):                               # nn.GRU default init U(-1/sqrt(H), 1/sqrt(H))
            for n, shape in (("weight_ih", (3 * Hs, Hs)), ("weight_hh", (3 * Hs, Hs)), ("bias_ih", (3 * Hs,)), ("bias_hh", (3 * Hs,))):
                P[e + f"rnn_layer.{n}_l0{sfx}"] = _u(rs, shape, 1 / np.sqrt(Hs))
        P[e + "projection_layer.linear_layer.weight"] = _u(rs, (E, 2 * Hs), np.sqrt(6.0 / (2 * Hs + E)))
        P[e + "projection_layer.linear_layer.bias"] = _u(rs, (E,), 1 / np.sqrt(2 * Hs))
    elif with_style:
        E = style_embed  # = 2*Z with use_vae (modules.py:283)
        e = "style_encoder.encoder."
        xav = lambda co, ci, k, gain: gain * np.sqrt(6.0 / (ci * k + co * k))
        P[e + "convs.0.conv.weight"] = _u(rs, (style_hidden, P_IN, 3), xav(style_hidden, P_IN, 3, np.sqrt(2)))
        P[e + "convs.0.conv.bias"] = _u(rs, (style_hidden,), 1 / np.sqrt(P_IN * 3))
        P[e + "convs.2.weight"] = (1 + 0.1 * rs.randn(style_hidden)).astype(np.float32)
        P[e + "convs.2.bias"] = (0.1 * rs.randn(style_hidden)).astype(np.float32)
        P[e + "convs.4.conv.weight"] = _u(rs, (E, style_hidden, 3), xav(E, style_hidden, 3, np.sqrt(2)))
        P[e + "convs.4.conv.bias"] = _u(rs, (E,), 1 / np.sqrt(style_hidden * 3))
        P[e + "convs.6.weight"] = (1 + 0.1 * rs.randn(E)).astype(np.float32)
        P[e + "convs.6.bias"] = (0.1 * rs.randn(E)).astype(np.float32)
        a = e + "blocks.0.attention."
        P[a + "multi_head_attention.in_proj_weight"] = _u(rs, (3 * E, E), np.sqrt(6.0 / (4 * E)))
        P[a + "multi_head_attention.in_proj_bias"] = (0.02 * rs.randn(3 * E)).astype(np.float32)
        P[a + "multi_head_attention.out_proj.weight"] = _u(rs, (E, E), 1 / np.sqrt(E))
        P[a + "multi_head_attention.out_proj.bias"] = (0.02 * rs.randn(E)).astype(np.float32)
        P[a + "layer_norm.weight"] = (1 + 0.1 * rs.randn(E)).astype(np.float32)
        P[a + "layer_norm.bias"] = (0.1 * rs.randn(E)).astype(np.float32)
        f = e + "blocks.0.feed_forward."
        P[f + "convs.0.conv.weight"] = _u(rs, (E, E, 3), xav(E, E, 3, np.sqrt(2)))
        P[f + "convs.0.conv.bias"] = _u(rs, (E,), 1 / np.sqrt(E * 3))
        P[f + "convs.2.conv.weight"] = _u(rs, (E, E, 3), xav(E, E, 3, 1.0))
        P[f + "convs.2.conv.bias"] = _u(rs, (E,), 1 / np.sqrt(E * 3))
        P[f + "layer_norm.weight"] = (1 + 0.1 * rs.randn(E)).astype(np.float32)
        P[f + "layer_norm.bias"] = (0.1 * rs.randn(E)).astype(np.float32)
    if rnn_cond == "film":
        P = {k: v for k, v in P.items() if not k.startswith(d)}
        P.update(_film_decoder_params(H, S, Z, seed))
    return P


def _film_decoder_params(H, S, Z, seed):
    """RecurrentDecoderFiLM (modules.py:188-212): LinearNorm predictors (xavier-uniform weights), nn.Linear / nn.GRU default scales."""
    rs = np.random.RandomState(seed + 7919)
    d = "decoder.recurrent_decoder."
    A, kb = P_IN + S, 1 / np.sqrt(H)
    P = {}
    for n in ("gammas", "betas"):
        P[d + n + "_predictor.linear_layer.weight"] = _u(rs, (2 * H, Z), np.sqrt(6.0 / (Z + 2 * H)))
        P[d + n + "_predictor.linear_layer.bias"] = _u(rs, (2 * H,), 1 / np.sqrt(Z))
    P[d + "layer0.weight"] = _u(rs, (H, A), 1 / np.sqrt(A))
    P[d + "layer0.bias"] = _u(rs, (H,), 1 / np.sqrt(A))
    P[d + "layer1.weight_ih_l0"] = _u(rs, (3 * H, A + H), kb)
    P[d + "layer1.weight_hh_l0"] = _u(rs, (3 * H, H), kb)
    P[d + "layer1.bias_ih_l0"] = _u(rs, (3 * H,), kb)
    P[d + "layer1.bias_hh_l0"] = _u(rs, (3 * H,), kb)
    P[d + "layer1.weight_ih_l1"] = _u(rs, (3 * H, H), kb)
    P[d + "layer1.weight_hh_l1"] = _u(rs, (3 * H, H), kb)
    P[d + "layer1.bias_ih_l1"] = _u(rs, (3 * H,), kb)
    P[d + "layer1.bias_hh_l1"] = _u(rs, (3 * H,), kb)
    P[d + "layer2.weight"] = _u(rs, (H, H), kb)
    P[d + "layer2.bias"] = _u(rs, (H,), kb)
    P[d + "layer3.weight"] = _u(rs, (P_OUT, H), kb)
    P[d + "layer3.bias"] = _u(rs, (P_OUT,), kb)
    return P


def _orthonormal_xy(rs, shape):
    """Random rotation-matrix x/y axes, shape [..., 2, 3] (data_pipeline.py:175-177 layout)."""
    x = rs.randn(*shape, 3)
    y = rs.randn(*shape, 3)
    x /= np.linalg.norm(x, axis=-1, keepdims=True)
    y -= np.sum(x * y, axis=-1, keepdims=True) * x
    y /= np.linalg.norm(y, axis=-1, keepdims=True)
    return np.stack([x, y], axis=-2)


def make_pose_windows(B, T, seed=1234, stats=None):
    """W_* training windows [B,T,...] with realistic scales (SURVEY.md §8d):
    channel-wise mu_in + sigma_in*N(0,1) de-vectorised; unit root quaternions with w>0;
    orthonormal ltxy; gaze target = root_pos + 100*unit vector (data_pipeline.py:124-127)."""
    st = stats or load_stats()
    rs = np.random.RandomState(seed)
    mu = st["anim_input_mean"].astype(np.float64)
    sd = st["anim_input_std"].astype(np.float64)
    v = mu[None, None, :P_OUT] + sd[None, None, :P_OUT] * rs.randn(B, T, P_OUT) * 0.5
    o = 6
    root_vel, root_vrt = v[..., 0:3], v[..., 3:6]
    lpos = v[..., o:o + NJ * 3].reshape(B, T, NJ, 3)
    ltxy = _orthonormal_xy(rs, (B, T, NJ))
    lvel = v[..., o + NJ * 9:o + NJ * 12].reshape(B, T, NJ, 3)
    lvrt = v[..., o + NJ * 12:o + NJ * 15].reshape(B, T, NJ, 3)
    q = rs.randn(B, T, 4)
    q[..., 0] = np.abs(q[..., 0]) + 1.0
    q /= np.linalg.norm(q, axis=-1, keepdims=True)
    root_pos = np.cumsum(rs.randn(B, T, 3) * 0.5, axis=1) * np.array([1.0, 0.0, 1.0])
    g = rs.randn(B, 1, 3)
    g /= np.linalg.norm(g, axis=-1, keepdims=True)
    gaze_pos = root_pos[:, :1] + 100.0 * g + rs.randn(B, T, 3) * 2.0
    f = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(root_pos=f(root_pos), root_rot=f(q), root_vel=f(root_vel), root_vrt=f(root_vrt), lpos=f(lpos),
                ltxy=f(ltxy), lvel=f(lvel), lvrt=f(lvrt), gaze_pos=f(gaze_pos))


def make_audio_features(B, T, seed=1234, stats=None):
    """[B,T,81] = mu_audio + sigma_audio*N(0,1) (raw, un-normalised features)."""
    st = stats or load_stats()
    rs = np.random.RandomState(seed + 1)
    return (st["audio_input_mean"][None, None] + float(st["audio_input_std"]) * rs.randn(B, T, N_AUDIO)).astype(np.float32)


def make_style_example(B, T_ex, seed=1234, stats=None):
    """[B,T_ex,1134] raw style example, gaze slot zero before normalisation (dataset.py:194-197)."""
    st = stats or load_stats()
    rs = np.random.RandomState(seed + 2)
    x = st["anim_input_mean"][None, None].astype(np.float64) + st["anim_input_std"][None, None] * rs.randn(B, T_ex, P_IN) * 0.5
    x[..., P_OUT:] = 0.0
    return x.astype(np.float32)


def make_waveforms(n_clips, n_samples=160000, seed=1234):
    """[N, n_samples] f32: 0.05*N(0,1) + a few sinusoids (so mel bins are not flat), clipped to [-1,1]."""
    rs = np.random.RandomState(seed + 3)
    t = np.arange(n_samples, dtype=np.float64) / 16000.0
    out = np.empty((n_clips, n_samples), dtype=np.float32)
    for i in range(n_clips):
        x = 0.05 * rs.randn(n_samples)
        for _ in range(3):
            f0 = rs.uniform(80.0, 4000.0)
            x += rs.uniform(0.02, 0.2) * np.sin(2 * np.pi * f0 * t + rs.uniform(0, 6.28))
        x *= 0.5 + 0.5 * np.sin(2 * np.pi * rs.uniform(0.2, 2.0) * t) ** 2
        out[i] = np.clip(x, -1.0, 1.0)
    return out
