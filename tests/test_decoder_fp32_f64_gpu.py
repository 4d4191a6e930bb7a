"""The fp32 decoder engine (the default engine, and the only one for the FiLM decoder and for hidden sizes outside the tensor-core rule)
against the float64 oracle (model_oracle / film_oracle through autograd) at the bounds of oracle/fp32_oracle.py:
forward max-abs <= FP32_FWD_TOL * max(1, max|ref|) per pose-channel group; every parameter gradient, dSpeech and dStyle max-abs <=
FP32_GEMM_GRAD_TOL * max|ref| in GEMM mode 1 (split-bf16 products) and FP32_GRAD_TOL * max|ref| in GEMM mode 0.
tests/test_decoder_fp32_oracle_cpu.py shows that float32 arithmetic meets those bounds with 4x headroom and that small kernel faults
break them.

Covered: the forward at every accepted hidden size; the geometry the kernels branch on (units per CTA U = 4 / 8, fewer k-chunks than
warps, one and several 32-sample batch tiles, label style Z = 9, S + Z = 256); the training shape with both weight-gradient paths
(split-bf16 GEMMs and the SIMT kernels, in GEMM mode 0 and as the mode-1 fallback when the histories do not fit the scratch buffer);
the split-K workspace at the very end of the scratch buffer; the largest batch one call takes and the error one sample more gets; the
FiLM decoder.  Every case prints its worst error and its ratio to the bound."""
import math

import numpy as np
import pytest
import torch

from oracle import film_oracle as fo
from oracle import fp32_oracle as f3
from oracle import model_oracle as mo
from tests._util import NAMES, ensure_built, make_decoder, run_with_grads, stats_tensors, tt

pytestmark = pytest.mark.gpu

STATS = ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


@pytest.fixture
def ops(dev):
    """zeggs_b200.ops on the fp32 engine; the engine and the GEMM mode are restored afterwards."""
    from zeggs_b200 import ops
    prev, prev_mode = ops.DECODER_ENGINE, ops.GEMM_MODE
    ops.set_decoder_engine("fp32")
    yield ops
    ops.set_decoder_engine(prev)
    ops.set_gemm_mode(prev_mode)


@pytest.fixture
def private_lane(ops, dev):
    """-> install(buf, scratch_bytes): a lane whose context uses the caller's scratch tensor and scratch size; removed afterwards."""
    from zeggs_b200 import _lib
    name = "fp32_oracle_test"
    key = (str(dev), name)

    def install(buf, scratch_bytes):
        ops._scratch[key] = buf
        ops._ctx[key] = _lib.Ctx(scratch=buf.data_ptr(), scratch_bytes=int(scratch_bytes), gemm_mode=ops.GEMM_MODE, fast_wgrad=0)
        return ops.lane(name)
    yield install
    torch.cuda.synchronize()
    ops._scratch.pop(key, None)
    ops._ctx.pop(key, None)


def _case(H, B, T, Z, seed, film=False, S=64):
    from zeggs_b200 import synth
    P = synth.make_params(H=H, S=S, Z=Z, seed=seed, with_style=False, rnn_cond="film" if film else "normal")
    win = tt(synth.make_pose_windows(B, T, seed=seed))
    rs = np.random.RandomState(seed)
    speech = torch.from_numpy((rs.randn(B, T, S) * 0.5).astype(np.float32))
    style = torch.from_numpy(rs.randn(B, T, Z).astype(np.float32))
    cot = [torch.from_numpy(rs.randn(*win[n].shape).astype(np.float32)) for n in NAMES]
    return P, win, speech, style, cot


def _decoder(P, H, S, Z, film, dev):
    if not film:
        return make_decoder(P, H, S=S, Z=Z, device=dev)
    from zeggs_b200 import modules
    dec = modules.Decoder(1134, 1131, S, Z, H, 2, rnn_cond="film")
    dec.load_state_dict({k[len("decoder."):]: torch.from_numpy(v) for k, v in P.items() if k.startswith("decoder.")})
    return dec.to(dev).eval()


def _run_gpu(dev, P, win, speech, style, cot, film=False, grads=True):
    """The decoder module on the fp32 engine -> (8 outputs, {name: gradient of sum(out * cot)} or None), on the CPU."""
    H = P["decoder.recurrent_decoder.layer0.weight"].shape[0]
    S, Z = speech.shape[-1], style.shape[-1]
    st = stats_tensors(dev)
    dec = _decoder(P, H, S, Z, film, dev)
    args = [win[n][:, 0].to(dev) for n in NAMES] + [win["gaze_pos"].to(dev)]
    stats = [st[k] for k in STATS]
    if not grads:
        with torch.no_grad():
            out = dec(*args, speech.to(dev), style.to(dev), st["parents"], *stats, st["dt"])
        torch.cuda.synchronize()
        return [o.cpu() for o in out], None
    dec.train()
    sp, sy = speech.to(dev).requires_grad_(True), style.to(dev).requires_grad_(True)
    out = dec(*args, sp, sy, st["parents"], *stats, st["dt"])
    named = dict(dec.named_parameters())
    keys = sorted("decoder." + k for k in named)
    g = torch.autograd.grad(sum((o * c.to(dev)).sum() for o, c in zip(out, cot)), [named[k[len("decoder."):]] for k in keys] + [sp, sy])
    torch.cuda.synchronize()
    return [o.detach().cpu() for o in out], {k: v.cpu() for k, v in zip(keys + ["speech", "style"], g)}


def _reference(P, win, speech, style, cot, film=False, grads=True):
    """float64 oracle: outputs, and with grads=True the autograd gradients of sum(out * cot)."""
    fn = fo.decoder_forward_film if film else mo.decoder_forward
    if grads:
        return run_with_grads(fn, P, win, speech, style, cot)
    st = stats_tensors()
    Pd = {k: torch.from_numpy(v).double() for k, v in P.items() if k.startswith("decoder.")}
    with torch.no_grad():
        out = fn(Pd, *[win[n][:, 0].double() for n in NAMES], win["gaze_pos"].double(), speech.double(), style.double(),
                 *[st[k].double() for k in STATS], st["dt"])
    return list(out), None


def _check(tag, got, ref, g_got=None, g_ref=None, gemm_mode=1):
    """Assert the bounds; print the worst forward and gradient errors and their ratio to the bound."""
    bad = []
    for n, o in zip(NAMES, got):
        assert torch.isfinite(o).all(), (tag, n)
    fe = f3.forward_errors(got, ref)
    n, e = max(fe.items(), key=lambda kv: kv[1])
    msg = f"  [{tag}] forward worst {n} {e:.3e} ({e / f3.FP32_FWD_TOL:.3f} of bound)"
    bad += [(k, v) for k, v in fe.items() if not v <= f3.FP32_FWD_TOL]
    if g_got is not None:
        gtol = f3.FP32_GEMM_GRAD_TOL if gemm_mode == 1 else f3.FP32_GRAD_TOL
        assert set(g_got) == set(g_ref), set(g_got) ^ set(g_ref)
        ge = f3.grad_errors(g_got, g_ref)
        k, e = max(ge.items(), key=lambda kv: kv[1])
        msg += f"  gradient worst {k} {e:.3e} ({e / gtol:.3f} of bound)"
        bad += [(k, v) for k, v in ge.items() if not v <= gtol]
    print(msg)
    assert not bad, (tag, bad)


# ---------------------------------------------------------------------------------------------------------- every hidden size
@pytest.mark.parametrize("H", list(range(16, 1056 + 1, 16)))
def test_forward_every_hidden_size(dev, ops, H):
    case = _case(H, 3, 5, 64, seed=3000 + H)
    got, _ = _run_gpu(dev, *case, grads=False)
    ref, _ = _reference(*case, grads=False)
    _check(f"fwd H{H} B3 T5", got, ref)


# ---------------------------------------------------------------------------------------------------------- geometry edges
EDGE_H = (16, 48, 80, 208, 512, 528, 544, 1024, 1056)
EDGE_CASES = [(H, B, T, 64, 64) for H in EDGE_H for B in (1, 32, 33, 65) for T in (2, 17)] + \
             [(16, 33, 17, 9, 64), (528, 65, 17, 9, 64), (1056, 33, 17, 9, 64), (544, 33, 17, 192, 64)]


@pytest.mark.parametrize("H,B,T,Z,S", EDGE_CASES)
def test_geometry_edges_forward_backward(dev, ops, H, B, T, Z, S):
    """U = 4 up to H = 528 and U = 8 from 544 (528 and 1056 fill all 132 SMs); H <= 112 has fewer 16-row k-chunks than warps and
    H = 16 one; B = 33 / 65 run two / three batch tiles with a one-sample tail; Z = 9 is the label style; S + Z = 256 the widest
    conditioning input."""
    case = _case(H, B, T, Z, seed=4000 + H + B + T + Z, S=S)
    got, g = _run_gpu(dev, *case)
    ref, g_ref = _reference(*case)
    _check(f"H{H} B{B} T{T} S{S} Z{Z}", got, ref, g, g_ref)


# ---------------------------------------------------------------------------------------------------------- training shape
TRAIN = (1024, 32, 256)


def _hist_bytes(H, B, T, S, Z, lo=True):
    """Bytes of the bf16 copies of the 11 weight-gradient histories (wgrad_hists in csrc/decoder_bwd.cu): rows x T*nbt*32 bf16 each."""
    rows = 1131 + 4 * 3 * H + 4 * H + 1134 + S + Z
    return rows * T * math.ceil(B / 32) * 32 * 2 * (2 if lo else 1)


@pytest.fixture(scope="module")
def train_case():
    H, B, T = TRAIN
    case = _case(H, B, T, 64, seed=5150)
    return case, _reference(*case)


@pytest.mark.parametrize("path", ["gemm", "simt_mode0", "simt_fallback"])
def test_training_shape_both_weight_gradient_paths(dev, ops, private_lane, train_case, path):
    """B = 32, T = 256, H = 1024: forward and the full BPTT.  gemm: GEMM mode 1 with the default scratch, the weight gradients are
    split-bf16 tensor-core GEMMs; simt_mode0: GEMM mode 0, the SIMT kernels; simt_fallback: GEMM mode 1 on a lane whose scratch is one
    256-byte block short of the histories, so the weight gradients fall back to the SIMT kernels."""
    case, (ref, g_ref) = train_case
    H, B, T = TRAIN
    mode = 0 if path == "simt_mode0" else 1
    ops.set_gemm_mode(mode)
    if path == "simt_fallback":
        need = _hist_bytes(H, B, T, 64, 64)
        buf = torch.empty(need, dtype=torch.uint8, device=dev)
        with private_lane(buf, need - 256):
            got, g = _run_gpu(dev, *case)
    else:
        got, g = _run_gpu(dev, *case)
    _check(f"train shape H{H} B{B} T{T} {path}", got, ref, g, g_ref, gemm_mode=mode)


def test_splitk_workspace_at_the_end_of_the_scratch(dev, ops, private_lane):
    """The bf16 histories end 128 bytes past a 256-byte boundary (T * nbt = 17 is odd) and the scratch buffer ends 64 bytes behind
    them: the 256-aligned split-K workspace starts past the end, so there is no room for split-K partials.  The weight-gradient GEMMs
    (dW2: 9 output tiles, K = 512, a split-K shape) must still be right and write nothing behind the buffer: the test's own
    allocation continues for 16 MiB behind it, filled with a sentinel that must come back unchanged."""
    ops.set_gemm_mode(1)
    H, B, T, S, Z = 64, 32, 17, 64, 64
    need = _hist_bytes(H, B, T, S, Z)
    assert need % 256 == 128
    scratch = need + 64
    buf = torch.full((scratch + (16 << 20),), 0xA5, dtype=torch.uint8, device=dev)
    assert buf.data_ptr() % 256 == 0
    case = _case(H, B, T, Z, seed=6060, S=S)
    with private_lane(buf, scratch):
        got, g = _run_gpu(dev, *case)
    tail = buf[scratch:]
    changed = int((tail != 0xA5).sum())
    ref, g_ref = _reference(*case)
    _check(f"split-K edge H{H} B{B} T{T} (scratch = histories + 64 B)", got, ref, g, g_ref)
    print(f"  sentinel bytes changed behind the scratch buffer: {changed}")
    assert changed == 0


# ---------------------------------------------------------------------------------------------------------- batch limit
def _fwd_smem(U, nbt):
    """fwd_smem_bytes (csrc/decoder_fwd.cu): dynamic shared memory of the forward recurrence."""
    stg = 16 * 4 * (6 * U // 4) + 1024
    return (8 * 2 * stg + 8 * 6 * U * 32 + nbt * 3 * U * 32 + 6 * 32) * 4


def _bwd_smem(H, U, nbt):
    """bwd_smem_bytes (csrc/decoder_bwd.cu): dynamic shared memory of the BPTT recurrence."""
    n4b = math.ceil(max(9, math.ceil(1134 / (H // U))) / 16)
    stg = 16 * 16 + 1024
    return (8 * 2 * stg + 8 * 16 * 32 + 2 * nbt * U * 32 + nbt * n4b * 16 * 32 + nbt * 9 * 32 + nbt * 7 * 32) * 4


def _max_batch(smem_of, cap):
    nbt = 1
    while smem_of(nbt + 1) <= cap:
        nbt += 1
    assert smem_of(1) <= cap
    return 32 * nbt


@pytest.mark.parametrize("H", [16, 1056])
def test_largest_batch_and_one_more(dev, ops, H):
    """U = 4 at H = 16 (the BPTT stages 284 x_pose-gradient rows per CTA) and U = 8 at H = 1056: the largest batch whose shared memory
    fits runs and matches the oracle; one sample more is refused with a ZeggsError that names the limit -- for the backward at its
    limit and for the forward at its own."""
    from zeggs_b200 import _lib
    cap = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    U = f3.units_per_cta(H)
    b_fwd = _max_batch(lambda n: _fwd_smem(U, n), cap)
    b_bwd = _max_batch(lambda n: _bwd_smem(H, U, n), cap)
    print(f"  H{H} U{U}: largest batch forward {b_fwd}, backward {b_bwd} ({cap} bytes of shared memory per block)")
    assert b_bwd <= b_fwd
    case = _case(H, b_bwd, 2, 64, seed=7000 + H)
    got, g = _run_gpu(dev, *case)
    ref, g_ref = _reference(*case)
    _check(f"largest backward batch H{H} B{b_bwd} T2", got, ref, g, g_ref)
    with pytest.raises(_lib.ZeggsError, match=f"at most {b_bwd} samples"):
        _run_gpu(dev, *_case(H, b_bwd + 1, 2, 64, seed=7001 + H))
    case = _case(H, b_fwd, 2, 64, seed=7002 + H)
    got, _ = _run_gpu(dev, *case, grads=False)
    ref, _ = _reference(*case, grads=False)
    _check(f"largest forward batch H{H} B{b_fwd} T2", got, ref)
    with pytest.raises(_lib.ZeggsError, match=f"at most {b_fwd} samples"):
        _run_gpu(dev, *_case(H, b_fwd + 1, 2, 64, seed=7003 + H), grads=False)


# ---------------------------------------------------------------------------------------------------------- FiLM
@pytest.mark.parametrize("H", [16, 528, 544, 1056])
@pytest.mark.parametrize("B,T", [(1, 2), (1, 17), (33, 2), (33, 17)])
def test_film_forward_backward(dev, ops, H, B, T):
    case = _case(H, B, T, 64, seed=8000 + H + B + T, film=True)
    got, g = _run_gpu(dev, *case, film=True)
    ref, g_ref = _reference(*case, film=True)
    _check(f"film H{H} B{B} T{T}", got, ref, g, g_ref)


def test_film_training_shape_forward(dev, ops):
    H, B, T = TRAIN
    case = _case(H, B, T, 64, seed=8888, film=True)
    got, _ = _run_gpu(dev, *case, film=True, grads=False)
    ref, _ = _reference(*case, film=True, grads=False)
    _check(f"film train shape H{H} B{B} T{T}", got, ref)
