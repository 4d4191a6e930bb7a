"""Planner rule, inputs, float64 oracles, arithmetic restatements and modelled faults of the GEMM front end (`zeggs_gemm_f32_ctx` /
`gemm_f32_auto` in csrc/tc_gemm.cu, the SIMT kernels of csrc/gemm.cu and the wgmma kernel of csrc/tc_gemm.cu), shared by
tests/test_gemm_f64_cpu.py (no GPU: the bounds mean something) and tests/test_gemm_f64_gpu.py (the kernels meet them).

* `expected_path`: which arithmetic a product gets -- `simt`, `simt_n32`, `tc3` (split-bf16, three passes), `tc1` (one bf16 pass,
  mode-1 products of a fast_wgrad context), each tensor-core path with or without split-K -- restated from `plan_tc_operands` and the
  split rule of `tc_gemm_launch`, for a device of `sms` SMs.  `launches` is the `zeggs_launch_count()` delta of one call.
* Oracles (float64, torch, on any device): `oracle` = act(op(A) op(B) + bias) + C0; `matched` rounds the operands to bf16 first (the
  one-pass paths); `split3` is the three-pass scheme hi*hi + lo*hi + hi*lo without lo*lo.
* Bound, elementwise: |got - ref| <= tau_path(K) (S + |bias|) + 8u |ref| with S = |op(A)| |op(B)| in float64.  It scales with every row
  and column, so a small row or column cannot hide behind the largest element.  ELU and ReLU are 1-Lipschitz, so the pre-activation
  bound carries through them.  The last rounding of an accumulate (C + x) alone costs up to u |ref| where |C| dominates, so the
  relative term is 8u rather than 2u: 4x headroom at the worst rounding.
* `restate_simt` / `restate_tc`: the kernels' arithmetic in float64 holding float32 values -- the SIMT kernels as one fp32 FMA per k
  in k order; the tensor-core kernel as one fp32 accumulation per 16-wide k step and pass, rounded toward zero (the tensor cores'
  accumulator is not round-to-nearest; truncation is the pessimistic model), split-K partials summed in z order -- plus the
  modelled faults (FAULTS).
"""
import math
from collections import namedtuple

import torch

U = 2.0 ** -24                 # fp32 unit roundoff
TC_MIN_MACS = 4.0e6            # plan_tc_operands: smaller products stay on the SIMT kernel
TG_BM, TG_BK = 128, 64         # tensor-core tile rows, k-block depth
GRID_Y = 65535                 # CUDA's grid.y limit: row tiles per launch

# tau per path (tests/test_gemm_f64_cpu.py shows the restatements below meet it with >= 4x headroom):
#   fp32 accumulation: tau_acc(K) = u (4 sqrt(K) + 16) -- the probabilistic bound lambda sqrt(K) u of a K-term fp32 sum, plus the
#   roundings of the epilogue (bias, activation, accumulate) and the last rounding of the tensor cores' truncating accumulator;
#   split-bf16 operands: a product misses lo*lo and the residuals a - hi - lo, b - hi - lo, together <= 3 * 2^-16 |a b|.  Over K
#   products of random sign that averages down as 1/sqrt(K): eps3(K) = 2^-13 min(1, 4 / sqrt(K)).  At K <= 16 it is 2.7x the worst
#   case of one product, so the 4x headroom holds where a few products decide the element.
OLD_REL = 4e-5                 # the max|C|-relative check the earlier front-end tests used


def tau_acc(K):
    return U * (4.0 * math.sqrt(K) + 16.0)


def eps3(K):
    return 2.0 ** -13 * min(1.0, 4.0 / math.sqrt(K))


def tau(kind, K):
    """tau of a path: `simt` / `simt_n32` and `tc1` (against the bf16-matched oracle) are fp32 accumulation; `tc3` adds the split error."""
    return tau_acc(K) + (eps3(K) if kind == "tc3" else 0.0)


# ---------------------------------------------------------------------------------------------- planner
Ctx = namedtuple("Ctx", "gemm_mode scratch_bytes fast_wgrad")       # scratch_bytes None: no scratch


class Path(namedtuple("Path", "kind splits BN")):
    @property
    def name(self):
        return self.kind + (f"_splitk({self.splits})" if self.splits > 1 else "")

    def launches(self, M):
        """zeggs_launch_count() delta of one front-end call: the SIMT kernel once per slice of 65535 row tiles; the tensor cores two
        operand splits, one GEMM launch per slice and the split-K reduction."""
        if self.kind.startswith("simt"):
            return math.ceil(M / (GRID_Y * (128 if self.kind == "simt_n32" else 64)))
        return 2 + math.ceil(math.ceil(M / TG_BM) / GRID_Y) + (self.splits > 1)


def round_up(x, m):
    return (x + m - 1) // m * m


def carve_bytes(M, N, K, three):
    """plan_tc_operands' operand carve (Ah, Bh [, Al, Bl] of Kp = round_up(K, 8) bf16 each, every piece rounded up to 256 bytes) from a
    256-byte aligned scratch base."""
    Kp = round_up(K, 8)
    ab = round_up(M * Kp * 2, 256) + round_up(N * Kp * 2, 256)
    return ab * (2 if three else 1)


def simt_path(mode, M, N):
    return Path("simt_n32" if (N <= 32 and mode != 0 and M >= 128) else "simt", 1, 0)


def tc_splits(M, N, K, BN, sms, ws_bytes):
    """tc_gemm_launch's split count (ws_bytes None: no split-K workspace, as zeggs_tc_gemm_bf16)."""
    tiles = math.ceil(N / BN) * math.ceil(M / TG_BM)
    kblocks = math.ceil(K / TG_BK)
    splits = 1
    if ws_bytes is not None and tiles <= sms // 2 and kblocks >= 8:
        splits = min(max(1, sms // tiles), kblocks // 2)
        per = M * N * 4
        if splits * per > ws_bytes:
            splits = ws_bytes // per
        splits = max(splits, 1)
    kbs = math.ceil(kblocks / splits)
    return math.ceil(kblocks / kbs)


def tc_bn(three, N):
    return 256 if (not three and N >= 256) else 128


def expected_path(mode, M, N, K, ctx, sms):
    """The path zeggs_gemm_f32_ctx takes for this product under `ctx` on a device of `sms` SMs."""
    assert ctx.gemm_mode in (0, 1)
    three = not (mode == 1 and ctx.fast_wgrad)
    if ctx.gemm_mode == 0 or not ctx.scratch_bytes or M * N * K < TC_MIN_MACS:
        return simt_path(mode, M, N)
    carve = carve_bytes(M, N, K, three)
    if carve > ctx.scratch_bytes:
        return simt_path(mode, M, N)
    BN = tc_bn(three, N)
    return Path("tc3" if three else "tc1", tc_splits(M, N, K, BN, sms, ctx.scratch_bytes - carve), BN)


def bf16_entry_path(M, N, three):
    """zeggs_tc_gemm_bf16: the tensor-core kernel alone, no split-K workspace."""
    return Path("tc3" if three else "tc1", 1, tc_bn(three, N))


# ---------------------------------------------------------------------------------------------- inputs
def make_operands(mode, M, N, K, seed, dyn=False, device="cpu"):
    """Stored operands (A [M,K] or, mode 1, [K,M]; B [N,K] in mode 0, else [K,N]), bias [N] and C0 [M,N], fp32 randn.  `dyn`: rows
    of op(A) and columns of op(B) scaled by 10^U(-3, 3), so elements of C span twelve decades."""
    g = torch.Generator(device=device).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=device)
    A = rn(K, M) if mode == 1 else rn(M, K)
    B = rn(N, K) if mode == 0 else rn(K, N)
    bias, C0 = rn(N), rn(M, N)
    if dyn:
        sa = 10.0 ** (torch.rand(M, generator=g, device=device) * 6 - 3)
        sb = 10.0 ** (torch.rand(N, generator=g, device=device) * 6 - 3)
        A = A * (sa[None, :] if mode == 1 else sa[:, None])
        B = B * (sb[:, None] if mode == 0 else sb[None, :])
        C0 = C0 * sa[:, None] * sb[None, :]
    return A, B, bias, C0


def op_a(mode, A):
    """[M, K] view of the stored A."""
    return A.T if mode == 1 else A


def op_b(mode, B):
    """[K, N] view of the stored B."""
    return B.T if mode == 0 else B


def bf16(x):
    """round-to-nearest-even to bf16, as float64"""
    return x.float().to(torch.bfloat16).double()


def split_hi_lo(x):
    """the kernels' split: hi = bf16(x), lo = bf16(x - hi) (the fp32 difference is exact), as float64"""
    x = x.float()
    hi = x.to(torch.bfloat16)
    return hi.double(), (x - hi.float()).to(torch.bfloat16).double()


# ---------------------------------------------------------------------------------------------- oracles and bound
def _act64(x, act):
    if act == 1:
        return torch.where(x > 0, x, torch.expm1(x))
    if act == 2:
        return x.clamp_min(0.0)
    return x


def epilogue64(P, bias, act, C0):
    x = P + bias.double()[None, :] if bias is not None else P
    x = _act64(x, act)
    return x + C0.double() if C0 is not None else x


def oracle(mode, A, B, bias=None, act=0, C0=None):
    return epilogue64(op_a(mode, A).double() @ op_b(mode, B).double(), bias, act, C0)


def matched(mode, A, B, bias=None, act=0, C0=None):
    """float64 product of the bf16-rounded operands: what one bf16 pass computes exactly"""
    return epilogue64(bf16(op_a(mode, A)) @ bf16(op_b(mode, B)), bias, act, C0)


def split3(mode, A, B, bias=None, act=0, C0=None):
    """float64 emulation of the three-pass scheme: hi*hi + lo*hi + hi*lo"""
    ah, al = split_hi_lo(op_a(mode, A))
    bh, bl = split_hi_lo(op_b(mode, B))
    return epilogue64(ah @ bh + al @ bh + ah @ bl, bias, act, C0)


def scale(mode, A, B, bias=None):
    """S + |bias| of the bound: |op(A)| |op(B)| in float64"""
    S = op_a(mode, A).double().abs() @ op_b(mode, B).double().abs()
    return S + bias.double().abs()[None, :] if bias is not None else S


def ratio(got, ref, S, t):
    """elementwise |got - ref| / (t S + 8u |ref|), NaN -> inf: the worst value is the case's ratio to its bound"""
    r = (got.double() - ref).abs() / (t * S + 8 * U * ref.abs() + 1e-300)
    return torch.where(torch.isnan(r), torch.full_like(r, math.inf), r)


def old_check(got, ref):
    """the earlier tests' check: max|err| <= 4e-5 max|C|"""
    return float((got.double() - ref).abs().max()) <= OLD_REL * float(ref.abs().max())


# ---------------------------------------------------------------------------------------------- restatements and faults
FAULTS = {
    "lo_hi_dropped": "the lo*hi pass of the split-bf16 product is not issued",
    "k_tail_dropped": "the partial last k-block (K mod 64 rows of the contraction) never reaches the product",
    "m_tail_unwritten": "rows 64..127 of the last row tile (the second consumer warpgroup's) are not stored",
    "bias_twice": "the tile adds the bias to its split-K partial and the reduction adds it again",
    "accumulate_ignored": "accumulate = 1 overwrites C instead of adding to it",
    "act_before_bias": "the activation is applied before the bias is added",
    "splitk_partial_missing": "the reduction sums every split-K partial but the last",
    "mode1_lda_is_M": "mode 1 reads A[k][m] at k*M + m instead of k*lda + m",
    "n_tail_past_N": "the N-tail store writes one column past N (outside the output window)",
    "n32_last_chunk_dropped": "the n32 kernel drops its last 32-deep k chunk",
    "fast_wgrad_in_mode0": "fast_wgrad's one bf16 pass runs a mode-0 product",
}


def _rn32(x):
    return x.float().double()


def _rz32(x):
    """float64 -> float32 rounded toward zero, as float64"""
    r = x.float()
    over = r.double().abs() > x.abs()
    return torch.where(over, torch.nextafter(r, torch.zeros_like(r)), r).double()


def epilogue32(x, bias, act, C0, fault=None):
    """the kernels' fp32 epilogue: + bias, activation, + C (accumulate)"""
    if fault == "act_before_bias":
        x = _act32(x, act)
        return _rn32(x + bias.double()[None, :]) if bias is not None else x
    if bias is not None:
        x = _rn32(x + bias.double()[None, :])
    x = _act32(x, act)
    if C0 is not None and fault != "accumulate_ignored":
        x = _rn32(x + C0.double())
    return x


def _act32(x, act):
    if act == 1:
        return torch.where(x > 0, x, _rn32(torch.expm1(x)))
    return x.clamp_min(0.0) if act == 2 else x


def restate_simt(mode, A, B, bias=None, act=0, C0=None, fault=None, A_store=None):
    """sgemm_kernel / sgemm_n32_kernel: acc = fmaf(a_k, b_k, acc) for k = 0 .. K-1, then the epilogue.  `A_store` (mode 1): the
    contiguous [K, lda] buffer A is a view of, for the mode1_lda_is_M fault."""
    a, b = op_a(mode, A).double(), op_b(mode, B).double()
    M, K = a.shape
    if fault == "mode1_lda_is_M":
        a = A_store.reshape(-1)[: K * M].reshape(K, M).T.double()
    kend = K
    if fault == "n32_last_chunk_dropped":
        kend = (K - 1) // 32 * 32
    elif fault == "k_tail_dropped":
        kend = K // TG_BK * TG_BK
    acc = torch.zeros(M, b.shape[1], dtype=torch.float64)
    for k in range(kend):
        acc = _rn32(acc + a[:, k:k + 1] * b[k:k + 1, :])
    return epilogue32(acc, bias, act, C0, fault)


def restate_tc(mode, A, B, bias=None, act=0, C0=None, three=True, splits=1, fault=None):
    """tc_gemm_kernel (+ splitk_reduce_kernel): per 16-wide k step the pass(es) hi*hi [, lo*hi, hi*lo] each added to the fp32
    accumulator (rounded toward zero); with split-K, split z owns k-blocks [z kbs, (z+1) kbs) and the reduction sums the partials in z
    order from 0, then applies the epilogue."""
    a, b = op_a(mode, A), op_b(mode, B)
    if fault == "fast_wgrad_in_mode0":
        three = False
    M, K = a.shape
    N = b.shape[1]
    kblocks = math.ceil(K / TG_BK)
    Kpad = kblocks * TG_BK
    ah, al = split_hi_lo(a)
    bh, bl = split_hi_lo(b)
    pad = lambda x, dim: torch.nn.functional.pad(x, (0, Kpad - K) if dim == 1 else (0, 0, 0, Kpad - K))
    ah, al, bh, bl = pad(ah, 1), pad(al, 1), pad(bh, 0), pad(bl, 0)
    if fault == "k_tail_dropped":
        k_live = K // TG_BK * TG_BK
        ah[:, k_live:] = 0
    kbs = math.ceil(kblocks / splits)
    parts = []
    for z in range(splits):
        acc = torch.zeros(M, N, dtype=torch.float64)
        for ks in range(z * kbs * TG_BK, min((z + 1) * kbs, kblocks) * TG_BK, 16):
            s = slice(ks, ks + 16)
            acc = _rz32(acc + ah[:, s] @ bh[s, :])
            if three:
                if fault != "lo_hi_dropped":
                    acc = _rz32(acc + al[:, s] @ bh[s, :])
                acc = _rz32(acc + ah[:, s] @ bl[s, :])
        parts.append(acc)
    if splits == 1:
        return epilogue32(parts[0], bias, act, C0, fault)
    if fault == "bias_twice" and bias is not None:
        parts = [_rn32(p + bias.double()[None, :]) for p in parts]
    if fault == "splitk_partial_missing":
        parts = parts[:-1]
    x = torch.zeros(M, N, dtype=torch.float64)
    for p in parts:
        x = _rn32(x + p)
    return epilogue32(x, bias, act, C0, fault)


def m_tail_unwritten(out, M, fill=0.0):
    """rows 64..127 of the last row tile keep what the buffer held"""
    out = out.clone()
    last = (M - 1) // TG_BM * TG_BM
    if M - last > 64:
        out[last + 64:] = fill
    return out
