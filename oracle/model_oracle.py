"""CPU oracle (PyTorch fp32, functional) for the ZeroEGGS network hot path.

TEST INFRASTRUCTURE ONLY -- a restatement of the reference algorithm, used as the
checker in tests/, `__graft_entry__.smoke()` and bench.py's cpu_baseline / `--impl
reference` leg.  The product path (zeggs_b200.*) never imports this file and has no
CPU fallback.

Every function takes a flat dict `P` of tensors keyed by the REFERENCE state-dict names
(SURVEY.md §8b), prefixed "speech_encoder." / "style_encoder." / "decoder.", so the
shipped pickles' state dicts can be fed in directly.

Pinned: tests/test_oracle_vs_reference.py runs each function against the imported
reference modules (/root/reference/ZEGGS, when present: random-init AND the shipped v1
pickles); oracle/make_golden.py writes reference outputs to tests/golden/*.npz which
tests re-check without the reference tree.

Reference lines restated (relative to /root/reference/ZEGGS):
  modules.py:249-272   SpeechEncoder
  modules.py:289-304, 391-420, 445-481, 496-513, 533-557, 595-612, 643-651  StyleEncoder (attn, VAE)
  modules.py:230-243   CellStateEncoder
  modules.py:165-185   RecurrentDecoderNormal (nn.GRU, gate order r,z,n; b_hn inside r*(...))
  modules.py:677-742   vectorize_input / devectorize_output
  modules.py:47-162    Decoder.forward
  modules.py:745-789   KL weight annealing / compute_KL_div
  anim/tquat.py:5-32, 49-67, 93-106   quaternion helpers (w-first)
  anim/txform.py:10-34 xform_fk_vel / xform_orthogonalize_from_xy
  train.py:277-421     world-space transforms, FK, 17 L1 terms + KL, /18
  optimizers.py:31-99  RAdam
"""
import math

import torch
import torch.nn.functional as F

NJ = 75


# ----------------------------------------------------------------------------- quaternions
def quat_mul(x, y):  # tquat.py:5-15
    x0, x1, x2, x3 = x[..., 0:1], x[..., 1:2], x[..., 2:3], x[..., 3:4]
    y0, y1, y2, y3 = y[..., 0:1], y[..., 1:2], y[..., 2:3], y[..., 3:4]
    return torch.cat([
        y0 * x0 - y1 * x1 - y2 * x2 - y3 * x3,
        y0 * x1 + y1 * x0 - y2 * x3 + y3 * x2,
        y0 * x2 + y1 * x3 + y2 * x0 - y3 * x1,
        y0 * x3 - y1 * x2 + y2 * x1 + y3 * x0], dim=-1)


def quat_mul_vec(q, v):  # tquat.py:17-20
    t = 2.0 * torch.cross(q[..., 1:], v, dim=-1)
    return v + q[..., 0:1] * t + torch.cross(q[..., 1:], t, dim=-1)


def quat_inv(q):  # tquat.py:22-24
    return q * torch.tensor([1.0, -1.0, -1.0, -1.0], dtype=q.dtype)


def quat_inv_mul_vec(q, v):  # tquat.py:30-32
    return quat_mul_vec(quat_inv(q), v)


def quat_normalize(x, eps=1e-5):  # tquat.py:49-51
    return x / (torch.norm(x, dim=-1, keepdim=True) + eps)


def quat_to_xform(x):  # tquat.py:53-67
    qw, qx, qy, qz = x[..., 0:1], x[..., 1:2], x[..., 2:3], x[..., 3:4]
    x2, y2, z2 = qx + qx, qy + qy, qz + qz
    xx, yy, wx = qx * x2, qy * y2, qw * x2
    xy, yz, wy = qx * y2, qy * z2, qw * y2
    xz, zz, wz = qx * z2, qz * z2, qw * z2
    return torch.cat([
        torch.cat([1.0 - (yy + zz), xy - wz, xz + wy], dim=-1)[..., None, :],
        torch.cat([xy + wz, 1.0 - (xx + zz), yz - wx], dim=-1)[..., None, :],
        torch.cat([xz - wy, yz + wx, 1.0 - (xx + yy)], dim=-1)[..., None, :]], dim=-2)


def quat_exp(x, eps=1e-5):  # tquat.py:93-98
    halfangle = torch.norm(x, dim=-1, keepdim=True)
    return torch.where(
        halfangle < eps,
        quat_normalize(torch.cat([torch.ones_like(halfangle), x], dim=-1)),
        torch.cat([torch.cos(halfangle), x * torch.sinc(halfangle / math.pi)], dim=-1))


def quat_from_helical(x, eps=1e-5):  # tquat.py:104-106
    return quat_exp(x / 2.0, eps)


# ----------------------------------------------------------------------------- xforms
def xform_orthogonalize_from_xy(xy, eps=1e-10):  # txform.py:23-34 (cross taken on the last dim)
    xaxis = xy[..., 0:1, :]
    zaxis = torch.cross(xaxis, xy[..., 1:2, :], dim=-1)
    yaxis = torch.cross(zaxis, xaxis, dim=-1)
    out = torch.cat([
        xaxis / (torch.norm(xaxis, 2, dim=-1)[..., None] + eps),
        yaxis / (torch.norm(yaxis, 2, dim=-1)[..., None] + eps),
        zaxis / (torch.norm(zaxis, 2, dim=-1)[..., None] + eps)], dim=-2)
    return out.transpose(-1, -2)


def xform_fk_vel(lxform, lpos, lvrt, lvel, parents):  # txform.py:10-20
    gr, gp, gt, gv = [lxform[..., :1, :, :]], [lpos[..., :1, :]], [lvrt[..., :1, :]], [lvel[..., :1, :]]
    for i in range(1, len(parents)):
        p = int(parents[i])
        rp = torch.matmul(gr[p], lpos[..., i:i + 1, :][..., None])[..., 0]
        gp.append(gp[p] + rp)
        gr.append(torch.matmul(gr[p], lxform[..., i:i + 1, :, :]))
        gt.append(gt[p] + torch.matmul(gr[p], lvrt[..., i:i + 1, :][..., None])[..., 0])
        gv.append(gv[p] + torch.matmul(gr[p], lvel[..., i:i + 1, :][..., None])[..., 0]
                  + torch.cross(gt[p], rp, dim=-1))
    return torch.cat(gr, dim=-3), torch.cat(gp, dim=-2), torch.cat(gt, dim=-2), torch.cat(gv, dim=-2)


def normalize_vec(x, eps=1e-8):  # modules.py:672-674
    return x / (torch.norm(x, dim=-1, keepdim=True) + eps)


# ----------------------------------------------------------------------------- SpeechEncoder
def speech_encoder(P, x, masks=None, prefix="speech_encoder."):
    """modules.py:265-272. x[B,T,81] (already (x-mean)/std) -> [B,T,64].
    masks: optional (m0[B,64,T], m1[B,64,T]) dropout multipliers (0 or 1/(1-p)), train mode."""
    g = lambda k: P[prefix + k]
    h = x.transpose(1, 2)
    h = F.elu(F.conv1d(h, g("layer0.weight"), g("layer0.bias")))               # k=1
    if masks is not None:
        h = h * masks[0]
    k = g("layer1.weight").shape[-1]
    h = F.pad(h, (k // 2, k - 1 - k // 2), mode="replicate")                    # padding='same', replicate
    h = F.elu(F.conv1d(h, g("layer1.weight"), g("layer1.bias")))
    if masks is not None:
        h = h * masks[1]
    h = h.transpose(1, 2)
    return F.elu(F.linear(h, g("layer2.weight"), g("layer2.bias")))


# ----------------------------------------------------------------------------- StyleEncoder
def positional_encoding(T, E, timestep=10000.0):
    """modules.py:445-481 for equal lengths: rows 0..T-1 of the sinusoid table."""
    pos = torch.arange(0, T, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, E, 2).float() * (-math.log(timestep) / E))
    pe = torch.zeros(T, E)
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


def _conv_k3(x, w, b):  # ConvNorm1D modules.py:643-651, zero padding 1; x[B,T,C]
    return F.conv1d(x.transpose(1, 2), w, b, padding=1).transpose(1, 2)


def style_encoder_attn(P, x, masks=None, prefix="style_encoder.", nheads=4, return_internals=False):
    """modules.py:391-420. x[B,T,1134] (normalised) -> pooled [B,E].
    masks: optional dict of dropout multipliers (train mode):
      'c1'[B,T,512] 'c2'[B,T,E] (p=.2), 'attn'[B,nheads,T,T] (p=.1, on softmax probabilities),
      'ao'[B,T,E] (p=.1), 'ff'[B,T,E] (p=.1)."""
    g = lambda k: P[prefix + "encoder." + k]
    m = masks or {}
    B, T, _ = x.shape
    h = F.relu(_conv_k3(x, g("convs.0.conv.weight"), g("convs.0.conv.bias")))
    h = F.layer_norm(h, (h.shape[-1],), g("convs.2.weight"), g("convs.2.bias"))
    if "c1" in m:
        h = h * m["c1"]
    h = F.relu(_conv_k3(h, g("convs.4.conv.weight"), g("convs.4.conv.bias")))
    E = h.shape[-1]
    h = F.layer_norm(h, (E,), g("convs.6.weight"), g("convs.6.bias"))
    if "c2" in m:
        h = h * m["c2"]
    x0 = h + positional_encoding(T, E)[None]                                     # :410 (mask all False)
    # nn.MultiheadAttention (modules.py:529, 544-550): q scaled by 1/sqrt(d_head)
    a = "blocks.0.attention."
    qkv = F.linear(x0, g(a + "multi_head_attention.in_proj_weight"), g(a + "multi_head_attention.in_proj_bias"))
    q, k, v = qkv.split(E, dim=-1)
    d = E // nheads
    q = q.reshape(B, T, nheads, d).transpose(1, 2)
    k = k.reshape(B, T, nheads, d).transpose(1, 2)
    v = v.reshape(B, T, nheads, d).transpose(1, 2)
    s = torch.matmul(q * (1.0 / math.sqrt(d)), k.transpose(-1, -2))
    p = torch.softmax(s, dim=-1)
    if "attn" in m:
        p = p * m["attn"]
    o = torch.matmul(p, v).transpose(1, 2).reshape(B, T, E)
    o = F.linear(o, g(a + "multi_head_attention.out_proj.weight"), g(a + "multi_head_attention.out_proj.bias"))
    if "ao" in m:
        o = o * m["ao"]
    x1 = F.layer_norm(o + x0, (E,), g(a + "layer_norm.weight"), g(a + "layer_norm.bias"))   # :555
    f = "blocks.0.feed_forward."
    y = F.relu(_conv_k3(x1, g(f + "convs.0.conv.weight"), g(f + "convs.0.conv.bias")))
    y = _conv_k3(y, g(f + "convs.2.conv.weight"), g(f + "convs.2.conv.bias"))
    if "ff" in m:
        y = y * m["ff"]
    x2 = F.layer_norm(y + x1, (E,), g(f + "layer_norm.weight"), g(f + "layer_norm.bias"))   # :603
    pooled = torch.sum(x2, dim=1) / float(T)                                    # :416-418
    if return_internals:
        return pooled, dict(x0=x0, x1=x1, x2=x2)
    return pooled


def style_encoder(P, x, eps=None, temperature=1.0, masks=None, prefix="style_encoder.", use_vae=True):
    """modules.py:289-304 -> (z, mu, logvar).  eps[B,Z] is the injected N(0,1) sample
    (reference: torch.randn_like, :299); eps=None -> zeros (z = mu)."""
    out = style_encoder_attn(P, x, masks, prefix)
    if not use_vae:
        return out, None, None
    Z = out.shape[1] // 2
    mu, logvar = out[:, :Z], out[:, Z:]
    std = torch.exp(0.5 * logvar) / temperature
    if eps is None:
        eps = torch.zeros_like(std)
    return mu + eps * std, mu, logvar


# ----------------------------------------------------------------------------- Decoder
def vectorize_input(root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt, gaze_pos, in_mean, in_std):
    # modules.py:677-713
    B = lpos.shape[0]
    gaze_dir = quat_inv_mul_vec(root_rot, gaze_pos - root_pos)
    enc = torch.cat([root_vel.reshape(B, -1), root_vrt.reshape(B, -1), lpos.reshape(B, -1), ltxy.reshape(B, -1),
                     lvel.reshape(B, -1), lvrt.reshape(B, -1), gaze_dir.reshape(B, -1)], dim=1)
    return (enc - in_mean) / in_std


def devectorize_output(pred, root_pos, root_rot, dt, out_mean, out_std, nj=NJ):
    # modules.py:716-742
    B = pred.shape[0]
    pred = pred * out_std + out_mean
    vel = pred[:, 0:3]
    vrt = pred[:, 3:6]
    lpos = pred[:, 6:6 + nj * 3].reshape(B, nj, 3)
    ltxy = pred[:, 6 + nj * 3:6 + nj * 9].reshape(B, nj, 2, 3)
    lvel = pred[:, 6 + nj * 9:6 + nj * 12].reshape(B, nj, 3)
    lvrt = pred[:, 6 + nj * 12:6 + nj * 15].reshape(B, nj, 3)
    new_pos = quat_mul_vec(root_rot, vel * dt) + root_pos
    new_rot = quat_mul(quat_from_helical(quat_mul_vec(root_rot, vrt * dt)), root_rot)
    return new_pos, new_rot, vel, vrt, lpos, ltxy, lvel, lvrt


def cell_state_encoder(P, pose, style, prefix="decoder.cell_state_encoder."):
    # modules.py:238-243 -> h[2,B,H]
    g = lambda k: P[prefix + k]
    h = F.elu(F.linear(torch.cat([pose, style], dim=-1), g("layer0.weight"), g("layer0.bias")))
    h = F.elu(F.linear(h, g("layer1.weight"), g("layer1.bias")))
    o = F.linear(h, g("layer2.weight"), g("layer2.bias"))
    return o.reshape(o.shape[0], 2, -1).swapaxes(0, 1).contiguous()


def gru_cell(x, h, w_ih, w_hh, b_ih, b_hh):
    """One nn.GRU layer, one step (PyTorch gate order r,z,n; b_hn inside r*(...))."""
    H = h.shape[-1]
    gi = F.linear(x, w_ih, b_ih)
    gh = F.linear(h, w_hh, b_hh)
    r = torch.sigmoid(gi[:, :H] + gh[:, :H])
    z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
    n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
    return (1.0 - z) * n + z * h


def recurrent_decoder_step(P, pose, speech, style, state, prefix="decoder.recurrent_decoder."):
    """modules.py:179-185.  state[2,B,H] -> (y[B,1131], new_state[2,B,H])."""
    g = lambda k: P[prefix + k]
    u = torch.cat([pose, speech, style], dim=-1)
    a = F.elu(F.linear(u, g("layer0.weight"), g("layer0.bias")))
    v = torch.cat([a, u], dim=-1)
    h0 = gru_cell(v, state[0], g("layer1.weight_ih_l0"), g("layer1.weight_hh_l0"),
                  g("layer1.bias_ih_l0"), g("layer1.bias_hh_l0"))
    h1 = gru_cell(h0, state[1], g("layer1.weight_ih_l1"), g("layer1.weight_hh_l1"),
                  g("layer1.bias_ih_l1"), g("layer1.bias_hh_l1"))
    y = F.linear(h1, g("layer2.weight"), g("layer2.bias"))
    return y, torch.stack([h0, h1], dim=0)


def decoder_forward(P, root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt,
                    gaze_pos, speech, style, in_mean, in_std, out_mean, out_std, dt, return_internals=False):
    """modules.py:47-162.  First-frame pose (8 tensors [B,...]), gaze_pos[B,T,3], speech[B,T,S],
    style[B,T,Z] -> 8-tuple with a time axis (frame 0 = the given pose)."""
    T = speech.shape[1]
    O = [[root_pos], [root_rot], [root_vel], [root_vrt], [lpos], [ltxy], [lvel], [lvrt]]
    x0 = vectorize_input(root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt, gaze_pos[:, 0], in_mean, in_std)
    state = cell_state_encoder(P, x0, style[:, 0])
    ys, states = [], [state]
    for i in range(1, T):
        pose = vectorize_input(O[0][-1], O[1][-1], O[2][-1], O[3][-1], O[4][-1], O[5][-1], O[6][-1], O[7][-1],
                               gaze_pos[:, i], in_mean, in_std)
        y, state = recurrent_decoder_step(P, pose, speech[:, i], style[:, i], state)
        new = devectorize_output(y, O[0][-1], O[1][-1], dt, out_mean, out_std, lpos.shape[1])
        for k in range(8):
            O[k].append(new[k])
        if return_internals:
            ys.append(y)
            states.append(state)
    out = tuple(torch.stack(o, dim=1) for o in O)
    if return_internals:
        return out, dict(y=torch.stack(ys, 1) if ys else None, states=torch.stack(states, 0), x0=x0)
    return out


# ----------------------------------------------------------------------------- losses (train.py)
def kl_weight(iteration, center=7500, rate=0.005, threshold=0.2):
    # modules.py:745-761, 784-788
    return min(1.0 / (1.0 + math.exp(-rate * (iteration - center))), threshold)


def compute_kl_div(mu, logvar, iteration):
    # modules.py:764-789
    kl = -0.5 * torch.mean(1 + logvar - mu.pow(2) - logvar.exp(), dim=1)
    return torch.mean(kl), kl_weight(iteration)


LOSS_NAMES = ["root_pos", "root_rot", "root_vel", "root_vrt", "lpos", "lrot", "lvel", "lvrt",
              "cpos", "crot", "cvel", "cvrt", "ldvl", "ldvt", "cdvl", "cdvt", "gaze"]


def _world_space(root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt, parents):
    """train.py:277-330 for one of O_* / W_* -> dict of world/character space tensors."""
    lmat = xform_orthogonalize_from_xy(ltxy)
    vel = torch.cat((quat_mul_vec(root_rot[:, 0:1], root_vel[:, 0:1]),
                     quat_mul_vec(root_rot[:, :-1], root_vel[:, 1:])), dim=1)          # :281-286
    vrt = torch.cat((quat_mul_vec(root_rot[:, 0:1], root_vrt[:, 0:1]),
                     quat_mul_vec(root_rot[:, :-1], root_vrt[:, 1:])), dim=1)
    rp0 = quat_mul_vec(root_rot, lpos[:, :, 0])
    lpos_0 = rp0 + root_pos                                                            # :296
    lmat_0 = torch.matmul(quat_to_xform(root_rot), lmat[:, :, 0])                      # :297
    lvel_0 = vel + quat_mul_vec(root_rot, lvel[:, :, 0]) + torch.cross(vrt, rp0, dim=-1)   # :298-302
    lvrt_0 = vrt + quat_mul_vec(root_rot, lvrt[:, :, 0])                               # :303
    lpos_w = torch.cat((lpos_0.unsqueeze(2), lpos[:, :, 1:]), dim=2)
    lmat_w = torch.cat((lmat_0.unsqueeze(2), lmat[:, :, 1:]), dim=2)
    lvel_w = torch.cat((lvel_0.unsqueeze(2), lvel[:, :, 1:]), dim=2)
    lvrt_w = torch.cat((lvrt_0.unsqueeze(2), lvrt[:, :, 1:]), dim=2)
    cmat, cpos, cvrt, cvel = xform_fk_vel(lmat_w, lpos_w, lvrt_w, lvel_w, parents)     # :325-330
    return dict(root_vel=vel, root_vrt=vrt, lpos=lpos_w, lvel=lvel_w, lvrt=lvrt_w,
                cmat=cmat, cpos=cpos, cvrt=cvrt, cvel=cvel, root_mat=quat_to_xform(root_rot))


def train_losses(O, W, gaze_pos, parents, dt, mu=None, logvar=None, iteration=0):
    """train.py:277-421.  O, W: 8-tuples (root_pos, root_rot, root_vel, root_vrt, lpos, ltxy, lvel, lvrt),
    each [B,T,...].  Returns (loss, dict of the 17 terms + kl)."""
    o = _world_space(*O, parents)
    w = _world_space(*W, parents)
    O_root_pos, O_root_rot, O_ltxy = O[0], O[1], O[5]
    W_root_pos, W_root_rot, W_ltxy = W[0], W[1], W[5]
    W_gaze_dir = quat_inv_mul_vec(W_root_rot, normalize_vec(gaze_pos - W_root_pos))    # :336
    O_gaze_dir = quat_inv_mul_vec(O_root_rot, normalize_vec(gaze_pos - O_root_pos))    # :337
    m = lambda s, a, b: torch.mean(torch.abs(s * (a - b)))
    dv = lambda s, a, b: torch.mean(torch.abs(s * ((a[:, 1:] - a[:, :-1]) / dt - (b[:, 1:] - b[:, :-1]) / dt)))
    L = {}
    L["root_pos"] = m(0.1, O_root_pos, W_root_pos)
    L["root_rot"] = m(10.0, o["root_mat"], w["root_mat"])
    L["root_vel"] = m(0.1, o["root_vel"], w["root_vel"])
    L["root_vrt"] = m(5.0, o["root_vrt"], w["root_vrt"])
    L["lpos"] = m(15.0, o["lpos"], w["lpos"])
    L["lrot"] = m(15.0, O_ltxy, W_ltxy)
    L["lvel"] = m(10.0, o["lvel"], w["lvel"])
    L["lvrt"] = m(7.0, o["lvrt"], w["lvrt"])
    L["cpos"] = m(0.1, o["cpos"], w["cpos"])
    L["crot"] = m(3.0, o["cmat"], w["cmat"])
    L["cvel"] = m(0.06, o["cvel"], w["cvel"])
    L["cvrt"] = m(1.25, o["cvrt"], w["cvrt"])
    L["ldvl"] = dv(7.0, o["lpos"], w["lpos"])
    L["ldvt"] = dv(8.0, O_ltxy, W_ltxy)
    L["cdvl"] = dv(0.06, o["cpos"], w["cpos"])
    L["cdvt"] = dv(1.25, o["cmat"], w["cmat"])
    L["gaze"] = m(10.0, O_gaze_dir, W_gaze_dir)
    total = sum(L[k] for k in LOSS_NAMES)
    if mu is not None and logvar is not None:
        kl, kw = compute_kl_div(mu, logvar, iteration)
        L["kl_div"] = kw * kl
        total = total + L["kl_div"]
    return total / 18.0, L


# static weight of each of the 17 terms (train.py:340-395)
LOSS_WEIGHTS = dict(root_pos=0.1, root_rot=10.0, root_vel=0.1, root_vrt=5.0, lpos=15.0, lrot=15.0, lvel=10.0, lvrt=7.0,
                    cpos=0.1, crot=3.0, cvel=0.06, cvrt=1.25, ldvl=7.0, ldvt=8.0, cdvl=0.06, cdvt=1.25, gaze=10.0)
DIFF_TERMS = ("ldvl", "ldvt", "cdvl", "cdvt")


def loss_residuals(O, W, gaze_pos, parents, dt):
    """The unweighted residuals whose absolute means `train_losses` weights, keyed by term name: term k is
    LOSS_WEIGHTS[k] * mean(|R[k]|).  Every residual is [B, T', ...] with T' = T for the 13 direct terms (root_rot = root
    matrix, lrot = raw two-axis ltxy, crot = FK matrix) and T' = T - 1 for the four frame-difference terms, whose index t
    is the difference between frames t + 1 and t.  Works in the dtype of the inputs."""
    o = _world_space(*O, parents)
    w = _world_space(*W, parents)
    O_gaze = quat_inv_mul_vec(O[1], normalize_vec(gaze_pos - O[0]))
    W_gaze = quat_inv_mul_vec(W[1], normalize_vec(gaze_pos - W[0]))
    dv = lambda a, b: (a[:, 1:] - a[:, :-1]) / dt - (b[:, 1:] - b[:, :-1]) / dt
    R = dict(root_pos=O[0] - W[0], root_rot=o["root_mat"] - w["root_mat"], root_vel=o["root_vel"] - w["root_vel"],
             root_vrt=o["root_vrt"] - w["root_vrt"], lpos=o["lpos"] - w["lpos"], lrot=O[5] - W[5], lvel=o["lvel"] - w["lvel"],
             lvrt=o["lvrt"] - w["lvrt"], cpos=o["cpos"] - w["cpos"], crot=o["cmat"] - w["cmat"], cvel=o["cvel"] - w["cvel"],
             cvrt=o["cvrt"] - w["cvrt"], ldvl=dv(o["lpos"], w["lpos"]), ldvt=dv(O[5], W[5]), cdvl=dv(o["cpos"], w["cpos"]),
             cdvt=dv(o["cmat"], w["cmat"]), gaze=O_gaze - W_gaze)
    return R


# ----------------------------------------------------------------------------- RAdam
def radam_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-5):
    """optimizers.py:31-99, one parameter tensor, weight_decay=0, degenerated_to_sgd=True.
    Updates p, m, v in place; `step` is the 1-based step count AFTER the increment."""
    v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
    m.mul_(beta1).add_(g, alpha=1 - beta1)
    beta2_t = beta2 ** step
    n_max = 2 / (1 - beta2) - 1
    n_sma = n_max - 2 * step * beta2_t / (1 - beta2_t)
    if n_sma >= 5:
        step_size = math.sqrt((1 - beta2_t) * (n_sma - 4) / (n_max - 4) * (n_sma - 2) / n_sma * n_max / (n_max - 2)) \
            / (1 - beta1 ** step)
        p.addcdiv_(m, v.sqrt().add_(eps), value=-step_size * lr)
    else:
        step_size = 1.0 / (1 - beta1 ** step)
        p.add_(m, alpha=-step_size * lr)
    return p
