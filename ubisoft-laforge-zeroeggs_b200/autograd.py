"""torch.autograd wiring for the C-ABI forward/backward pairs (plumbing only).  The bodies live in ops.*_fwd / ops.*_bwd, which
TrainStep also calls directly (explicit backward, no autograd engine in the training step)."""
import torch

from . import ops


class DecoderWindowFn(torch.autograd.Function):
    """(Y, root_pos, root_rot) = decoder window; backward = zeggs_decoder_window_bwd (full BPTT)."""

    @staticmethod
    def forward(ctx, dec, root_pos0, root_rot0, pose0, gaze_pos, speech, style, in_mean, in_std, out_mean, out_std,
                dt, *weights):
        Y, rp, rq, state = ops.decoder_window_forward(dec, root_pos0, root_rot0, pose0, gaze_pos, speech, style,
                                                      (in_mean, in_std, out_mean, out_std), dt, save=True)
        ctx.dec = dec
        ctx.state = state
        ctx.need_cond = (speech.requires_grad, style.requires_grad)
        return Y, rp, rq

    @staticmethod
    def backward(ctx, dY, dRp, dRq):
        grads, dSpeech, dStyle = ops.decoder_window_backward(ctx.dec, ctx.state, dY, dRp, dRq)
        ctx.state = None
        return (None, None, None, None, None, dSpeech if ctx.need_cond[0] else None, dStyle if ctx.need_cond[1] else None,
                None, None, None, None, None) + tuple(grads)


class SpeechEncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, enc, x, masks, *weights):
        y, ctx.state = ops.speech_encoder_fwd(enc, x, masks)
        return y

    @staticmethod
    def backward(ctx, dy):
        grads = ops.speech_encoder_bwd(ctx.state, dy)
        ctx.state = None
        return (None, None, None) + tuple(grads)


class StyleEncoderFn(torch.autograd.Function):
    """Outputs (z, mu, logvar) with the VAE, z alone without it; either encoder type."""

    @staticmethod
    def forward(ctx, enc, x, eps, masks, temperature, *weights):
        outs, ctx.state = ops.style_encoder_fwd(enc, x, eps, masks, temperature)
        return tuple(outs) if outs[1] is not None else outs[0]

    @staticmethod
    def backward(ctx, dz, dmu=None, dlv=None):
        grads = ops.style_encoder_bwd(ctx.state, dz, dmu, dlv)
        ctx.state = None
        return (None, None, None, None, None) + tuple(grads)


class TrainLossFn(torch.autograd.Function):
    """loss = train.py:277-421 evaluated (and differentiated) by zeggs_loss_fwd_bwd in the forward call."""

    @staticmethod
    def forward(ctx, Y, rp, rq, WY, Wrp, Wrq, gaze, parents_i32, dt, mu, logvar, kl_weight, terms_out, unit_grad=False, kl_weight_dev=None):
        loss, ctx.grads = ops.loss_fwd_bwd(Y, rp, rq, WY, Wrp, Wrq, gaze, parents_i32, dt, mu, logvar, kl_weight, terms_out, kl_weight_dev)
        ctx.unit_grad = bool(unit_grad)     # the caller promises loss.backward() with the implicit gradient 1
        return loss

    @staticmethod
    def backward(ctx, g):
        dY, dRp, dRq, dmu, dlv = ctx.grads
        ctx.grads = None
        s = (lambda t: t) if ctx.unit_grad else (lambda t: None if t is None else t * g)
        return (s(dY), s(dRp), s(dRq), None, None, None, None, None, None, s(dmu), s(dlv), None, None, None, None)
