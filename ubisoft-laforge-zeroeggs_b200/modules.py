"""`modules`-compatible network classes backed by the sm_90a kernels in libzeggs_b200.so.

Drop-in for ZEGGS/modules.py: same class names, constructor arguments, forward signatures and
state-dict keys (SURVEY.md §8b), so `load_state_dict()` of the shipped checkpoints works and the
reference's `train.py` / `generate.py` can run unchanged with this module registered as
`sys.modules["modules"]` (see INTEGRATION.md).  The parameter containers are ordinary
`nn.Linear / nn.GRU / nn.Conv1d / nn.LayerNorm / nn.MultiheadAttention` objects (that is what fixes
the key names); their own forward() is never called -- every forward here goes through the C ABI
(csrc/*.cu).  CUDA only: there is no CPU fallback.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from . import ops

NJ = 75
P_IN = 1134
P_OUT = 1131


# ===============================================================================================
#                                            Decoder
# ===============================================================================================
class RecurrentDecoderNormal(nn.Module):
    """Parameter container of modules.py:165-185 (keys layer0.*, layer1.weight_ih_l0..., layer2.*)."""

    def __init__(self, pose_input_size, speech_size, style_size, output_size, hidden_size, num_rnn_layers):
        super().__init__()
        all_input_size = pose_input_size + speech_size + style_size
        self.layer0 = nn.Linear(all_input_size, hidden_size)
        self.layer1 = nn.GRU(all_input_size + hidden_size, hidden_size, num_rnn_layers, batch_first=True)
        self.layer2 = nn.Linear(hidden_size, output_size)


class CellStateEncoder(nn.Module):
    """Parameter container of modules.py:230-243."""

    def __init__(self, input_size, hidden_size, num_rnn_layers):
        super().__init__()
        self.num_rnn_layers = num_rnn_layers
        self.layer0 = nn.Linear(input_size, hidden_size)
        self.layer1 = nn.Linear(hidden_size, hidden_size)
        self.layer2 = nn.Linear(hidden_size, hidden_size * num_rnn_layers)


class Decoder(nn.Module):
    """modules.py:11-162.  forward() = one launch sequence of zeggs_decoder_window_fwd (+ _bwd under autograd)."""

    def __init__(self, pose_input_size, pose_output_size, speech_encoding_size, style_encoding_size,
                 hidden_size, num_rnn_layers, rnn_cond="normal"):
        super().__init__()
        if rnn_cond != "normal":
            raise _lib.ZeggsError("only rnn_cond='normal' is on the accelerated path (the shipped configs)")
        if num_rnn_layers != 2:
            raise _lib.ZeggsError("num_rnn_layers must be 2 (train.py:124-131 hard-codes it)")
        if pose_input_size != P_IN or pose_output_size != P_OUT:
            raise _lib.ZeggsError("pose layout must be the 75-joint 1134/1131 layout (modules.py:699-736)")
        self.recurrent_decoder = RecurrentDecoderNormal(
            pose_input_size, speech_encoding_size, style_encoding_size, pose_output_size, hidden_size, num_rnn_layers)
        self.cell_state_encoder = CellStateEncoder(pose_input_size + style_encoding_size, hidden_size, num_rnn_layers)

    # sizes are read off the parameters so that instances un-pickled from the reference's whole-module checkpoints
    # (generate.py:130-138; they carry no extra attributes) work unchanged
    @property
    def hidden_size(self):
        return self.recurrent_decoder.layer0.weight.shape[0]

    @property
    def style_encoding_size(self):
        return self.cell_state_encoder.layer0.weight.shape[1] - P_IN

    @property
    def speech_encoding_size(self):
        return self.recurrent_decoder.layer0.weight.shape[1] - P_IN - self.style_encoding_size

    def _weights(self):
        r, c = self.recurrent_decoder, self.cell_state_encoder
        return [r.layer0.weight, r.layer0.bias,
                r.layer1.weight_ih_l0, r.layer1.bias_ih_l0, r.layer1.weight_hh_l0, r.layer1.bias_hh_l0,
                r.layer1.weight_ih_l1, r.layer1.bias_ih_l1, r.layer1.weight_hh_l1, r.layer1.bias_hh_l1,
                r.layer2.weight, r.layer2.bias,
                c.layer0.weight, c.layer0.bias, c.layer1.weight, c.layer1.bias, c.layer2.weight, c.layer2.bias]

    def forward(self, Z_root_pos, Z_root_rot, Z_root_vel, Z_root_vrt, Z_lpos, Z_ltxy, Z_lvel, Z_lvrt,
                Z_gaze_pos, speech_encoding, style_encoding, parents, anim_input_mean, anim_input_std,
                anim_output_mean, anim_output_std, dt: float):
        B = speech_encoding.shape[0]
        pose0 = torch.cat([Z_root_vel.reshape(B, -1), Z_root_vrt.reshape(B, -1), Z_lpos.reshape(B, -1),
                           Z_ltxy.reshape(B, -1), Z_lvel.reshape(B, -1), Z_lvrt.reshape(B, -1)], dim=1)
        Y, root_pos, root_rot = ops.decoder_window(
            self, Z_root_pos, Z_root_rot, pose0, Z_gaze_pos, speech_encoding, style_encoding,
            anim_input_mean, anim_input_std, anim_output_mean, anim_output_std, float(dt))
        return ops.split_pose(Y, root_pos, root_rot)

    def forward_packed(self, root_pos0, root_rot0, pose0, gaze_pos, speech_encoding, style_encoding,
                       anim_input_mean, anim_input_std, anim_output_mean, anim_output_std, dt: float):
        """Same window with the pose channels left packed ([B,T,1131] in the order of modules.py:731-736): what the fused
        loss consumes -- the trainer skips the split into 8 views and the re-concatenation (and their autograd)."""
        return ops.decoder_window(self, root_pos0, root_rot0, pose0, gaze_pos, speech_encoding, style_encoding,
                                  anim_input_mean, anim_input_std, anim_output_mean, anim_output_std, float(dt))


# ===============================================================================================
#                                  Small torch-side helpers kept for API parity
# ===============================================================================================
def normalize(x, eps: float = 1e-8):  # modules.py:672-674
    return x / (torch.norm(x, dim=-1, keepdim=True) + eps)


def generalized_logistic_function(x, center=0.0, B=1.0, A=0.0, K=1.0, C=1.0, Q=1.0, nu=1.0):  # modules.py:745-761
    return A + (K - A) / (C + Q * np.exp(-B * (x - center))) ** (1 / nu)


def compute_KL_div(mu, logvar, iteration):  # modules.py:764-789
    kl_div = torch.mean(-0.5 * torch.mean(1 + logvar - mu.pow(2) - logvar.exp(), dim=1))
    w = min(generalized_logistic_function(iteration, center=7500, B=0.005), 2e-1)
    return kl_div, w


# ===============================================================================================
#                                        Speech Encoder
# ===============================================================================================
class SpeechEncoder(nn.Module):
    """modules.py:249-272.  x[B,T,81] (normalised) -> [B,T,64] via zeggs_speech_enc_fwd/_bwd."""

    def __init__(self, input_size, hidden_size, output_size):
        super().__init__()
        self.layer0 = nn.Conv1d(input_size, hidden_size, kernel_size=1, padding="same", padding_mode="replicate")
        self.drop0 = nn.Dropout(p=0.2)
        self.layer1 = nn.Conv1d(hidden_size, output_size, kernel_size=31, padding="same", padding_mode="replicate")
        self.drop1 = nn.Dropout(p=0.2)
        self.layer2 = nn.Linear(output_size, output_size)

    def _weights(self):
        return [self.layer0.weight, self.layer0.bias, self.layer1.weight, self.layer1.bias,
                self.layer2.weight, self.layer2.bias]

    def forward(self, x, masks=None):
        """masks (testing hook): (m0[B,T,H], m1[B,T,O]) dropout multipliers; default: sampled in train mode."""
        return ops.speech_encoder(self, x, masks)


# ===============================================================================================
#                                        Style Encoder
# ===============================================================================================
class ConvNorm1D(nn.Module):
    """Parameter container of modules.py:615-651 (key `conv.*`)."""

    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=None, dilation=1, bias=True,
                 w_init_gain="linear"):
        super().__init__()
        self.conv = nn.Conv1d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=padding,
                              dilation=dilation, bias=bias)
        nn.init.xavier_uniform_(self.conv.weight, gain=nn.init.calculate_gain(w_init_gain))


class LinearNorm(nn.Module):
    def __init__(self, in_dim, out_dim, bias=True, w_init_gain="linear"):
        super().__init__()
        self.linear_layer = nn.Linear(in_dim, out_dim, bias=bias)
        nn.init.xavier_uniform_(self.linear_layer.weight, gain=nn.init.calculate_gain(w_init_gain))


class PositionalEncoding(nn.Module):
    """modules.py:445-481; only the table rows 0..T-1 are ever used (all lengths are equal, :399-403)."""

    def __init__(self, embed_dim, max_len=20000, timestep=10000.0):
        super().__init__()
        self.embed_dim = embed_dim
        self.timestep = timestep

    def table(self, T):
        pos = torch.arange(0, T, dtype=torch.float).unsqueeze(1)
        timestep = getattr(self, "timestep", 10000.0)   # absent on instances un-pickled from reference checkpoints
        div_term = torch.exp(torch.arange(0, self.embed_dim, 2).float() * (-np.log(timestep) / self.embed_dim))
        pe = torch.zeros(T, self.embed_dim)
        pe[:, 0::2] = torch.sin(pos * div_term)
        pe[:, 1::2] = torch.cos(pos * div_term)
        return pe


class MultiHeadAttention(nn.Module):
    def __init__(self, hidden_size):
        super().__init__()
        self.multi_head_attention = nn.MultiheadAttention(hidden_size, 4, 0.1)
        self.dropout = nn.Dropout(0.1)
        self.layer_norm = nn.LayerNorm(hidden_size)


class PositionWiseConvFF(nn.Module):
    def __init__(self, hidden_size):
        super().__init__()
        self.convs = nn.Sequential(
            ConvNorm1D(hidden_size, hidden_size, kernel_size=3, stride=1, padding=1, dilation=1, w_init_gain="relu"),
            nn.ReLU(),
            ConvNorm1D(hidden_size, hidden_size, kernel_size=3, stride=1, padding=1, dilation=1, w_init_gain="linear"),
            nn.Dropout(0.1))
        self.layer_norm = nn.LayerNorm(hidden_size)


class FFTBlock(nn.Module):
    def __init__(self, hidden_size):
        super().__init__()
        self.attention = MultiHeadAttention(hidden_size)
        self.feed_forward = PositionWiseConvFF(hidden_size)


class StyleEncoderAttn(nn.Module):
    """Parameter container of modules.py:346-389."""

    def __init__(self, input_size, hidden_size, style_embedding_size):
        super().__init__()
        self.pos_enc = PositionalEncoding(style_embedding_size)
        self.convs = nn.Sequential(
            ConvNorm1D(input_size, hidden_size, kernel_size=3, stride=1, padding=1, dilation=1, w_init_gain="relu"),
            nn.ReLU(), nn.LayerNorm(hidden_size), nn.Dropout(0.2),
            ConvNorm1D(hidden_size, style_embedding_size, kernel_size=3, stride=1, padding=1, dilation=1, w_init_gain="relu"),
            nn.ReLU(), nn.LayerNorm(style_embedding_size), nn.Dropout(0.2))
        self.blocks = nn.ModuleList([FFTBlock(style_embedding_size)])


class StyleEncoderGRU(nn.Module):
    """Parameter container of modules.py:307-343: conv k3 + ReLU twice, bidirectional one-layer GRU, projection of output[:, -1]."""

    def __init__(self, input_size, hidden_size, style_embedding_size):
        super().__init__()
        self.convs = nn.Sequential(
            ConvNorm1D(input_size, hidden_size, kernel_size=3, stride=1, padding=1, dilation=1, w_init_gain="relu"),
            nn.ReLU(),
            ConvNorm1D(hidden_size, hidden_size, kernel_size=3, stride=1, padding=1, dilation=1, w_init_gain="relu"),
            nn.ReLU())
        self.rnn_layer = nn.GRU(hidden_size, hidden_size, 1, batch_first=True, bidirectional=True)
        self.projection_layer = LinearNorm(hidden_size * 2, style_embedding_size, w_init_gain="linear")


class StyleEncoder(nn.Module):
    """modules.py:278-304.  forward(input[B,T_ex,1134], temprature) -> (z, mu, logvar), or (z, None, None) with use_vae=False.
    type 'attn' (StyleEncoderAttn) or 'gru' (StyleEncoderGRU); the encoder's output size is 2*style_embedding_size with the VAE,
    style_embedding_size without it.  The type is read off the encoder module, so whole-module pickles of the reference (which
    store no type) work unchanged."""

    def __init__(self, input_size, hidden_size, style_embedding_size, type="attn", use_vae=False):
        super().__init__()
        if type not in ("attn", "gru"):
            raise _lib.ZeggsError(f"unknown style encoder type {type!r} (modules.py:284-287 knows 'attn' and 'gru')")
        self.use_vae = use_vae
        self.style_embedding_size = style_embedding_size
        output_size = 2 * style_embedding_size if use_vae else style_embedding_size
        cls = StyleEncoderGRU if type == "gru" else StyleEncoderAttn
        self.encoder = cls(input_size, hidden_size, output_size)

    @property
    def encoder_type(self):
        return "gru" if isinstance(self.encoder, StyleEncoderGRU) else "attn"

    def _weights(self):
        e = self.encoder
        if self.encoder_type == "gru":
            r = e.rnn_layer
            return [e.convs[0].conv.weight, e.convs[0].conv.bias, e.convs[2].conv.weight, e.convs[2].conv.bias,
                    r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0,
                    r.weight_ih_l0_reverse, r.weight_hh_l0_reverse, r.bias_ih_l0_reverse, r.bias_hh_l0_reverse,
                    e.projection_layer.linear_layer.weight, e.projection_layer.linear_layer.bias]
        a, f = e.blocks[0].attention, e.blocks[0].feed_forward
        m = a.multi_head_attention
        return [e.convs[0].conv.weight, e.convs[0].conv.bias, e.convs[2].weight, e.convs[2].bias,
                e.convs[4].conv.weight, e.convs[4].conv.bias, e.convs[6].weight, e.convs[6].bias,
                m.in_proj_weight, m.in_proj_bias, m.out_proj.weight, m.out_proj.bias, a.layer_norm.weight, a.layer_norm.bias,
                f.convs[0].conv.weight, f.convs[0].conv.bias, f.convs[2].conv.weight, f.convs[2].conv.bias,
                f.layer_norm.weight, f.layer_norm.bias]

    def forward(self, input, temprature: float = 1.0, eps=None, masks=None):
        """eps / masks are testing hooks (injected N(0,1) sample and dropout multipliers)."""
        return ops.style_encoder(self, input, float(temprature), eps, masks)
