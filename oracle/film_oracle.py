"""CPU oracle of the FiLM-conditioned decoder (rnn_cond "film"), built from the blocks of oracle/model_oracle.py.

TEST INFRASTRUCTURE ONLY, like model_oracle.py.  Same conventions: a flat dict `P` keyed by the reference state-dict names.
Pinned to the unmodified reference by oracle/make_film_golden.py (tests/golden/train_film_*.npz).

Reference lines restated (relative to the reference's ZEGGS/):
  modules.py:188-227   RecurrentDecoderFiLM (gamma = 1 + predictor, FiLM after the ELU of layer0 and of layer2)
  modules.py:47-162    Decoder.forward (unchanged loop, the FiLM step in place of the normal one)
"""
import torch
import torch.nn.functional as F

from oracle.model_oracle import cell_state_encoder, devectorize_output, gru_cell, vectorize_input


def recurrent_decoder_film_step(P, pose, speech, style, state, prefix="decoder.recurrent_decoder."):
    """modules.py:214-227.  state[2,B,H] -> (y[B,1131], new_state[2,B,H])."""
    g = lambda k: P[prefix + k]
    H = g("layer0.weight").shape[0]
    gam = F.linear(style, g("gammas_predictor.linear_layer.weight"), g("gammas_predictor.linear_layer.bias")) + 1
    bet = F.linear(style, g("betas_predictor.linear_layer.weight"), g("betas_predictor.linear_layer.bias"))
    u = torch.cat([pose, speech], dim=-1)
    a = F.elu(F.linear(u, g("layer0.weight"), g("layer0.bias"))) * gam[:, :H] + bet[:, :H]
    v = torch.cat([a, u], dim=-1)
    h0 = gru_cell(v, state[0], g("layer1.weight_ih_l0"), g("layer1.weight_hh_l0"), g("layer1.bias_ih_l0"), g("layer1.bias_hh_l0"))
    h1 = gru_cell(h0, state[1], g("layer1.weight_ih_l1"), g("layer1.weight_hh_l1"), g("layer1.bias_ih_l1"), g("layer1.bias_hh_l1"))
    c = F.elu(F.linear(h1, g("layer2.weight"), g("layer2.bias"))) * gam[:, H:] + bet[:, H:]
    return F.linear(c, g("layer3.weight"), g("layer3.bias")), torch.stack([h0, h1], dim=0)


def decoder_forward_film(P, root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt,
                         gaze_pos, speech, style, in_mean, in_std, out_mean, out_std, dt):
    """modules.py:47-162 with rnn_cond="film": the arguments and the 8-tuple result of model_oracle.decoder_forward."""
    T = speech.shape[1]
    O = [[root_pos], [root_rot], [root_vel], [root_vrt], [lpos], [ltxy], [lvel], [lvrt]]
    x0 = vectorize_input(root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt, gaze_pos[:, 0], in_mean, in_std)
    state = cell_state_encoder(P, x0, style[:, 0])
    for i in range(1, T):
        pose = vectorize_input(O[0][-1], O[1][-1], O[2][-1], O[3][-1], O[4][-1], O[5][-1], O[6][-1], O[7][-1],
                               gaze_pos[:, i], in_mean, in_std)
        y, state = recurrent_decoder_film_step(P, pose, speech[:, i], style[:, i], state)
        new = devectorize_output(y, O[0][-1], O[1][-1], dt, out_mean, out_std, lpos.shape[1])
        for k in range(8):
            O[k].append(new[k])
    return tuple(torch.stack(o, dim=1) for o in O)
