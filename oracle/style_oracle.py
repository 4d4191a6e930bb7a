"""CPU oracle (PyTorch fp32, functional) of the StyleEncoder variants beyond the shipped attn + VAE: type 'gru' (StyleEncoderGRU)
and use_vae=False.

TEST INFRASTRUCTURE ONLY, like oracle/model_oracle.py, whose building blocks it uses.  Pinned against the unmodified reference
through tests/golden/style_gru.npz and tests/golden/train_gru_*.npz (oracle/make_style_golden.py).

Reference lines restated (relative to /root/reference/ZEGGS):
  modules.py:278-304   StyleEncoder (VAE on / off)
  modules.py:307-343   StyleEncoderGRU (bidirectional nn.GRU: both directions are scanned in full, no shortcut)
"""
import torch
import torch.nn.functional as F

from oracle.model_oracle import _conv_k3, gru_cell, style_encoder_attn


def gru_scan(x, w_ih, w_hh, b_ih, b_hh, reverse=False):
    """One direction of a one-layer nn.GRU over x[B,T,C] from h = 0 -> outputs [B,T,H] (position t holds the state after x[t])."""
    B, T, _ = x.shape
    h = x.new_zeros(B, w_hh.shape[1])
    out = [None] * T
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        h = gru_cell(x[:, t], h, w_ih, w_hh, b_ih, b_hh)
        out[t] = h
    return torch.stack(out, dim=1)


def style_encoder_gru(P, x, prefix="style_encoder."):
    """modules.py:307-343. x[B,T,1134] (normalised) -> projection of output[:, -1], [B,E]."""
    g = lambda k: P[prefix + "encoder." + k]
    h = F.relu(_conv_k3(x, g("convs.0.conv.weight"), g("convs.0.conv.bias")))
    h = F.relu(_conv_k3(h, g("convs.2.conv.weight"), g("convs.2.conv.bias")))
    w = lambda s: [g(f"rnn_layer.{n}_l0{s}") for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    out = torch.cat([gru_scan(h, *w("")), gru_scan(h, *w("_reverse"), reverse=True)], dim=-1)
    return F.linear(out[:, -1], g("projection_layer.linear_layer.weight"), g("projection_layer.linear_layer.bias"))


def style_encoder(P, x, eps=None, temperature=1.0, masks=None, prefix="style_encoder.", use_vae=True, type="attn"):
    """modules.py:289-304 -> (z, mu, logvar), or (z, None, None) with use_vae=False.  eps[B,Z] is the injected N(0,1) sample
    (reference: torch.randn_like, :299); eps=None -> zeros (z = mu).  type 'attn' or 'gru' (the GRU encoder has no dropout:
    masks apply to 'attn' only)."""
    out = style_encoder_gru(P, x, prefix) if type == "gru" else style_encoder_attn(P, x, masks, prefix)
    if not use_vae:
        return out, None, None
    Z = out.shape[1] // 2
    mu, logvar = out[:, :Z], out[:, Z:]
    std = torch.exp(0.5 * logvar) / temperature
    if eps is None:
        eps = torch.zeros_like(std)
    return mu + eps * std, mu, logvar
