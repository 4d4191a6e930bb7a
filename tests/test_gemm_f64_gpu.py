"""GPU: the GEMM front end (`zeggs_gemm_f32_ctx`, `zeggs_sgemm`, `zeggs_tc_gemm_bf16`) against float64 at every path, operand layout and
tile edge it accepts.  Planner rule, oracles and bounds: tests/_gemm_cases.py; tests/test_gemm_f64_cpu.py shows the bounds hold for
the kernels' arithmetic with >= 4x headroom and break under each modelled fault.  References are computed on the device in float64.

Every case checks four things:
* path: the zeggs_launch_count() delta equals the planner's (1 per SIMT slice; 3 on the tensor cores, 4 with split-K; 1 for
  zeggs_tc_gemm_bf16).  A one-pass product (64 elements or more, no bias) is also further than the three-pass bound from the
  unrounded float64 product;
* bound: |got - ref| <= tau_path(K) (S + |bias|) + 8u |ref| elementwise;
* guard band: C is a window of a larger buffer pre-filled with a NaN sentinel; every element outside the window is bitwise unchanged,
  none inside keeps the sentinel, and A and B are bitwise unchanged;
* determinism: a second call from the same state gives the same bits.

Cases: each GEMM mode on each path (SIMT by GEMM mode 0, by the 4e6 MAC threshold and by a scratch one byte short of the operand carve;
three passes with exactly the carve, with split-K on unlimited scratch and on scratch for two partials; one pass with N across the
BN = 256 switch); M, N and K tails; the n32 kernel; every epilogue on every path; the production stride patterns of the encoders, the
FiLM projections, the tensor-core engine's hoisted cond product and the FiLM backward; the shapes of the earlier front-end tests; and
products past 65535 row tiles (grid.y), which run in slices.  The 375 cases take 20 s on one H100 80GB HBM3 at 700 W; the worst
ratios to the bound there are in DESIGN.md section 2.
"""
import ctypes as C

import pytest
import torch

from tests import _gemm_cases as gc
from tests._util import ensure_built

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD          # a quiet NaN no kernel produces
MB = 1 << 20
P_IN = 1134


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


_scratch = {}


def _ctx(dev, gemm_mode, nbytes, fast):
    """a zeggs_ctx over the first `nbytes` of one 1536 MB scratch buffer (the size ops.ensure_scratch gives the main lane)"""
    from zeggs_b200 import _lib
    if "buf" not in _scratch:
        _scratch["buf"] = torch.empty(1536 * MB, dtype=torch.uint8, device=dev)
    buf = _scratch["buf"]
    assert nbytes <= buf.numel() and buf.data_ptr() % 256 == 0
    return _lib.Ctx(scratch=buf.data_ptr(), scratch_bytes=nbytes, gemm_mode=gemm_mode, fast_wgrad=fast)


def _spec(spec, mode, M, N, K):
    """(gemm_mode, scratch bytes, fast_wgrad) of a named context"""
    if spec in ("m0", "big", "fast"):
        return (0 if spec == "m0" else 1), 1536 * MB, int(spec == "fast")
    if spec in ("s256", "s256fast"):
        return 1, 256 * MB, int(spec == "s256fast")
    carve = gc.carve_bytes(M, N, K, True)
    return 1, {"carve": carve, "carve-1": carve - 1, "two": carve + 2 * M * N * 4}[spec], 0


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _i32(t):
    return t.view(torch.int32)


def _call(entry, ctx, mode, M, N, K, a, lda, b, ldb, bias, c, ldc, act, acc, a_lo=None, b_lo=None):
    """one product through an entry point -> zeggs_launch_count() delta"""
    from zeggs_b200 import _lib
    l = _lib.lib()
    n0 = l.zeggs_launch_count()
    if entry == "ctx":
        rc = l.zeggs_gemm_f32_ctx(C.addressof(ctx), mode, M, N, K, a, lda, b, ldb, bias, c, ldc, act, acc, _lib.stream_ptr())
    elif entry == "sgemm":
        rc = l.zeggs_sgemm(mode, M, N, K, a, lda, b, ldb, bias, c, ldc, act, acc, _lib.stream_ptr())
    else:
        rc = l.zeggs_tc_gemm_bf16(M, N, K, a, a_lo, lda, b, b_lo, ldb, bias, c, ldc, act, acc, _lib.stream_ptr())
    _lib.check(rc, entry)
    torch.cuda.synchronize()
    return l.zeggs_launch_count() - n0


def _embed(x, ld, off, g):
    """x [rows, cols] copied into a randn buffer at row stride ld and element offset off -> (buffer, view)"""
    rows, cols = x.shape
    flat = torch.randn(off + (rows - 1) * ld + cols + 7, generator=g, device=x.device)
    v = flat.as_strided((rows, cols), (ld, 1), off)
    v.copy_(x)
    return flat, v


def _run(dev, tag, entry, spec, mode, M, N, K, act=0, bias=False, acc=False, dyn=False, seed=0, lda=None, ldb=None, ldc=None,
         a_off=0, b_off=0, c_off=None, cbuf=None):
    """One checked product.  entry "ctx" (zeggs_gemm_f32_ctx under the context `spec`), "sgemm" (zeggs_sgemm) or "bf16"
    (zeggs_tc_gemm_bf16; spec "x3" or "x1", operands in mode-0 layout split by zeggs_split_bf16).  C is the [M, N] window at `c_off`,
    row stride `ldc`, of `cbuf` (a new sentinel-filled buffer by default; with `acc` the window of a given `cbuf` keeps its contents
    as C0).  -> (worst ratio to the bound, cbuf)"""
    from zeggs_b200 import ops
    A, B, bvec, C0 = gc.make_operands(mode, M, N, K, seed, dyn, device=dev)
    g = torch.Generator(device=dev).manual_seed(seed + 1)
    ldc = ldc or N + 5
    c_off = ldc + 3 if c_off is None else c_off
    if cbuf is None:
        cbuf = torch.empty(c_off + (M + 1) * ldc + 11, device=dev)
        _i32(cbuf).fill_(SENTINEL)
        if acc:
            cbuf.as_strided((M, N), (ldc, 1), c_off).copy_(C0)
    win = cbuf.as_strided((M, N), (ldc, 1), c_off)
    C0 = win.clone() if acc else None
    bias_t = bvec if bias else None
    bias_p = bvec.data_ptr() if bias else None
    lo_args = {}
    if entry == "bf16":
        three = spec == "x3"
        Ah, Al = ops.split_bf16(A, want_lo=three)
        Bh, Bl = ops.split_bf16(B, want_lo=three)
        for x, h, l in ((A, Ah, Al), (B, Bh, Bl)):        # zeggs_split_bf16 rounds as torch does, and zero-pads to Kp
            assert torch.equal(h[:, :K], x.to(torch.bfloat16)) and not h[:, K:].any()
            if three:
                assert torch.equal(l[:, :K], (x - h[:, :K].float()).to(torch.bfloat16)) and not l[:, K:].any()
        operands = [Ah, Al, Bh, Bl] if three else [Ah, Bh]
        args = (Ah.data_ptr(), Ah.stride(0), Bh.data_ptr(), Bh.stride(0))
        lo_args = dict(a_lo=Al.data_ptr() if three else None, b_lo=Bl.data_ptr() if three else None)
        path = gc.bf16_entry_path(M, N, three)
        ctx = None
    else:
        (ra, ca), (rb, cb) = A.shape, B.shape
        fa, A = _embed(A, lda or ca, a_off, g)
        fb, B = _embed(B, ldb or cb, b_off, g)
        operands = [fa, fb]
        args = (A.data_ptr(), lda or ca, B.data_ptr(), ldb or cb)
        if entry == "sgemm":
            path, ctx = gc.simt_path(mode, M, N), None
        else:
            gm, nbytes, fast = _spec(spec, mode, M, N, K)
            ctx = _ctx(dev, gm, nbytes, fast)
            path = gc.expected_path(mode, M, N, K, gc.Ctx(gm, nbytes, fast), _sms(dev))
    before = [x.clone() for x in operands]
    pre = cbuf.clone()
    launches = _call(entry, ctx, mode, M, N, K, args[0], args[1], args[2], args[3], bias_p, win.data_ptr(), ldc, act, int(acc), **lo_args)
    post = cbuf.clone()
    # guard band: outside the window nothing changed; inside no sentinel is left; the operands are untouched
    outside_pre, outside_post = pre.clone(), post.clone()
    outside_pre.as_strided((M, N), (ldc, 1), c_off).zero_()
    outside_post.as_strided((M, N), (ldc, 1), c_off).zero_()
    assert torch.equal(_i32(outside_pre), _i32(outside_post)), f"{tag}: elements outside the output window changed"
    assert not (_i32(win) == SENTINEL).any(), f"{tag}: output elements left unwritten"
    assert all(torch.equal(_i32(x), _i32(y)) for x, y in zip(before, operands)), f"{tag}: an operand was written"
    # bound
    t = gc.tau(path.kind, K)
    S = gc.scale(mode, A, B, bias_t)
    if path.kind == "tc1":
        ref = gc.matched(mode, A, B, bias_t, act, C0)
        far = float(gc.ratio(win, gc.oracle(mode, A, B, bias_t, act, C0), S, gc.tau("tc3", K)).max())
        if M * N >= 64 and not bias:
            assert far > 1.0, f"{tag}: within the three-pass bound of the unrounded product ({far:.3f}): not one bf16 pass"
    else:
        ref = gc.oracle(mode, A, B, bias_t, act, C0)
    worst = float(gc.ratio(win, ref, S, t).max())
    # determinism: the same call from the same state gives the same bits
    cbuf.copy_(pre)
    _call(entry, ctx, mode, M, N, K, args[0], args[1], args[2], args[3], bias_p, win.data_ptr(), ldc, act, int(acc), **lo_args)
    same = torch.equal(_i32(cbuf), _i32(post))
    print(f"  [{tag}] {entry} mode{mode} {M}x{N}x{K} act{act} bias{int(bias)} acc{int(acc)}{' dyn' if dyn else ''}: "
          f"{path.name}, {launches} launches, worst {worst:.3f} of its bound")
    want = path.launches(M) - (2 if entry == "bf16" else 0)        # zeggs_tc_gemm_bf16 is given split operands
    assert launches == want, f"{tag}: {launches} launches, {path.name} takes {want}"
    assert worst <= 1.0, f"{tag}: {worst:.3f} of the bound"
    assert same, f"{tag}: a second call gave different bits"
    return worst, cbuf


def _epi(i):
    """(act, bias, accumulate) of case i: all twelve combinations in turn"""
    return i % 3, bool((i // 3) % 2), bool((i // 6) % 2)


# ---------------------------------------------------------------------------------------------- each mode on each path
PATH_CASES = []
for _mode in (0, 1, 2):
    PATH_CASES += [
        ("m0", _mode, 200, 300, 1000),                 # GEMM mode 0: SIMT
        ("big", _mode, 160, 125, 200),                 # exactly 4e6 MACs: tensor cores
        ("big", _mode, 160, 125, 199),                 # one k less: SIMT
        ("carve-1", _mode, 256, 384, 512),             # scratch one byte short of the operand carve: SIMT
        ("carve", _mode, 256, 384, 512),               # exactly the carve: three passes, no room for split-K
        ("big", _mode, 32, 300, 4096),                 # split-K, unlimited scratch
        ("two", _mode, 64, 200, 2048),                 # split-K with scratch for exactly two partials
    ]
PATH_CASES += [("fast", 1, 64, n, 4096) for n in (255, 256, 257)]     # one pass with split-K, BN 128 / 256 / 256
PATH_CASES += [("fast", 1, 512, n, 384) for n in (255, 256, 257)]     # one pass, no split


@pytest.mark.parametrize("dyn", [False, True], ids=["randn", "dynrange"])
@pytest.mark.parametrize("spec,mode,M,N,K", PATH_CASES)
def test_each_mode_on_each_path(dev, spec, mode, M, N, K, dyn):
    act, bias, acc = _epi(M + N + K + mode)
    _run(dev, f"path {spec}", "ctx", spec, mode, M, N, K, act, bias, acc, dyn, seed=mode * 1000 + K)


def test_the_path_cases_reach_every_path(dev):
    sms = _sms(dev)
    names = set()
    for spec, mode, M, N, K in PATH_CASES:
        gm, nbytes, fast = _spec(spec, mode, M, N, K)
        p = gc.expected_path(mode, M, N, K, gc.Ctx(gm, nbytes, fast), sms)
        names.add(p.kind + ("_splitk" if p.splits > 1 else "") + ("_bn256" if p.BN == 256 else ""))
        if spec == "two":
            assert p.splits == 2
    assert names >= {"simt", "tc3", "tc3_splitk", "tc1", "tc1_bn256", "tc1_splitk", "tc1_splitk_bn256"}, names


# ---------------------------------------------------------------------------------------------- tails
TAIL_M = [1, 63, 64, 65, 127, 128, 129]
TAIL_N = [1, 17, 31, 32, 33, 127, 128, 129, 255, 256, 257]
TAIL_K = [1, 7, 8, 9, 63, 64, 65, 513, 12288]
TAIL_CASES = [(M, N, TAIL_K[(i + j) % len(TAIL_K)]) for i, M in enumerate(TAIL_M) for j, N in enumerate(TAIL_N)]


@pytest.mark.parametrize("M,N,K", TAIL_CASES)
def test_tails(dev, M, N, K):
    """every (M, N) tail pair, K cycling through its tails: the front end (SIMT or tensor cores, as the planner decides) and the
    tensor-core kernel itself in three passes and one"""
    i = TAIL_CASES.index((M, N, K))
    mode = i % 3
    act, bias, acc = _epi(i)
    _run(dev, "tail", "ctx", "big", mode, M, N, K, act, bias, acc, dyn=bool(i % 2), seed=i)
    for j, spec in enumerate(("x3", "x1")):
        act, bias, acc = _epi(i + 5 * j + 1)
        _run(dev, "tail", "bf16", spec, 0, M, N, K, act, bias, acc, dyn=bool((i + j) % 2), seed=i + 100 * j)


@pytest.mark.parametrize("K", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("M", [127, 128, 129])
@pytest.mark.parametrize("N", [1, 31, 32])
@pytest.mark.parametrize("mode", [1, 2])
def test_n32_kernel(dev, mode, N, M, K):
    act, bias, acc = _epi(mode + N + M + K)
    _run(dev, "n32", "ctx", "m0", mode, M, N, K, act, bias, acc, dyn=bool(K % 2), seed=M * K + N)


# ---------------------------------------------------------------------------------------------- every epilogue on every path
EPI_PATHS = {
    "simt": ("ctx", "m0", 0, 100, 70, 90),
    "simt_n32": ("ctx", "m0", 2, 256, 32, 100),
    "tc3": ("ctx", "big", 0, 256, 384, 384),
    "tc3_splitk": ("ctx", "big", 2, 32, 300, 4096),
    "tc1": ("ctx", "fast", 1, 512, 300, 384),
    "tc1_splitk": ("ctx", "fast", 1, 64, 300, 4096),
    "bf16_x1_bn256": ("bf16", "x1", 0, 130, 300, 192),
    "bf16_x1_bn128": ("bf16", "x1", 0, 130, 200, 192),
    "bf16_x3": ("bf16", "x3", 0, 130, 300, 192),
}


@pytest.mark.parametrize("acc", [False, True])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("name", list(EPI_PATHS))
def test_every_epilogue_on_every_path(dev, name, act, bias, acc):
    entry, spec, mode, M, N, K = EPI_PATHS[name]
    _run(dev, f"epilogue {name}", entry, spec, mode, M, N, K, act, bias, acc, dyn=acc, seed=act + 3 * bias)


# ---------------------------------------------------------------------------------------------- production stride patterns
@pytest.mark.parametrize("spec", ["m0", "big", "fast"])
def test_style_gru_reverse_cell_strides(dev, spec):
    """csrc/encoders.cu, GRU style encoder: the reverse cell reads h(T-1) of every sample at c2 + (T-1) H with row stride T H, and its
    input gradient accumulates into dc2 at the same place"""
    B, T, H = 33, 17, 256
    _run(dev, "gru rev fwd", "ctx", spec, 0, B, 3 * H, H, bias=True, seed=1, a_off=(T - 1) * H, lda=T * H, ldc=3 * H, c_off=0)
    _run(dev, "gru rev dW_ih_r", "ctx", spec, 1, 3 * H, H, B, seed=2, b_off=(T - 1) * H, ldb=T * H, ldc=H, c_off=0)
    _run(dev, "gru rev dc2", "ctx", spec, 2, B, H, 3 * H, acc=True, seed=3, ldc=T * H, c_off=(T - 1) * H)


@pytest.mark.parametrize("spec", ["m0", "big"])
def test_film_projections_fill_disjoint_column_halves(dev, spec):
    """csrc/decoder_fwd.cu: gamma - 1 and beta as two products into the column halves of GB [B T, 4H]; the second leaves the first
    half's bits alone and the first leaves the second half's sentinel alone"""
    BT, H, Z = 256, 256, 64
    _, buf = _run(dev, "film gamma", "ctx", spec, 0, BT, 2 * H, Z, bias=True, seed=4, ldc=4 * H, c_off=0)
    assert (_i32(buf[:BT * 4 * H].view(BT, 4 * H)[:, 2 * H:]) == SENTINEL).all()
    _run(dev, "film beta", "ctx", spec, 0, BT, 2 * H, Z, bias=True, seed=5, ldc=4 * H, c_off=2 * H, cbuf=buf)


@pytest.mark.parametrize("spec", ["m0", "big"])
def test_tc_engine_hoisted_cond_products(dev, spec):
    """csrc/decoder_fwd_tc.cu: S01 [(t, b)][4H] = cond rows . [W0[:, P_IN:] ; W_ih0[:, H + P_IN:]]^T + bfold, as a product into
    columns [0, H) with B at W0 + P_IN (row stride P_IN + C) and one into [H, 4H) with B at W_ih0 + H + P_IN (row stride H + P_IN + C)"""
    T, H, Cc = 16, 256, 128
    M, A_w = T * 32, P_IN + Cc
    _, buf = _run(dev, "cond W0", "ctx", spec, 0, M, H, Cc, bias=True, seed=6, b_off=P_IN, ldb=A_w, ldc=4 * H, c_off=0)
    _run(dev, "cond W_ih0", "ctx", spec, 0, M, 3 * H, Cc, bias=True, seed=7, b_off=H + P_IN, ldb=A_w + H, ldc=4 * H, c_off=H, cbuf=buf)


@pytest.mark.parametrize("spec", ["m0", "big", "fast"])
def test_film_backward_strides(dev, spec):
    """csrc/decoder_bwd.cu: dWg / dWb = DGB[:, 0:2H] / DGB[:, 2H:4H]^T style (lda = 4H), then dStyle = dG Wg + dBe Wb: the second
    product reads A at +2H and accumulates into the first one's output"""
    BT, H, Z = 512, 256, 64
    _run(dev, "film dWg", "ctx", spec, 1, 2 * H, Z, BT, seed=8, lda=4 * H, ldc=Z, c_off=0)
    _run(dev, "film dWb", "ctx", spec, 1, 2 * H, Z, BT, seed=9, a_off=2 * H, lda=4 * H, ldc=Z, c_off=0)
    _, buf = _run(dev, "film dStyle", "ctx", spec, 2, BT, Z, 2 * H, seed=10, lda=4 * H, ldc=Z, c_off=0)
    _run(dev, "film dStyle +=", "ctx", spec, 2, BT, Z, 2 * H, acc=True, seed=11, a_off=2 * H, lda=4 * H, ldc=Z, c_off=0, cbuf=buf)


# ---------------------------------------------------------------------------------------------- the earlier front-end tests' shapes
@pytest.mark.parametrize("M,N,K", [(7, 5, 3), (64, 64, 16), (130, 257, 1198), (32, 2048, 1024), (384, 32, 384), (200, 17, 100)])
def test_sgemm_entry(dev, M, N, K):
    _run(dev, "sgemm nt", "sgemm", None, 0, M, N, K, act=1, bias=True, seed=M * 1000 + N, ldc=N, c_off=0)
    _run(dev, "sgemm tn", "sgemm", None, 1, M, N, K, seed=M * 1000 + N + 1, ldc=N, c_off=0)


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 128, 256), (256, 384, 512), (200, 300, 1136), (3072, 2286, 1024),
                                   (1024, 1262, 4096), (130, 256, 192)])
def test_tc_gemm_bf16_entry(dev, M, N, K):
    for spec in ("x1", "x3"):
        _run(dev, f"tc_gemm_bf16 {spec}", "bf16", spec, 0, M, N, K, seed=M + N + K, ldc=N, c_off=0)


@pytest.mark.parametrize("mode,M,N,K", [(0, 300, 200, 1000), (1, 512, 3402, 1536), (2, 700, 260, 129), (0, 12288 // 8, 512, 3402),
                                        (0, 32, 512, 3402), (1, 128, 384, 12288), (2, 32, 1198, 2048), (1, 64, 64, 12288)])
def test_front_end_default_context_shapes(dev, mode, M, N, K):
    """the GEMM-mode-1 context ops.ensure_scratch makes for the main lane (1536 MB, fast_wgrad off); the last four split K"""
    _run(dev, "front end", "ctx", "big", mode, M, N, K, seed=mode * 7 + M, ldc=N, c_off=0)


def test_front_end_splitk_epilogue(dev):
    _run(dev, "split-K epilogue", "ctx", "big", 0, 32, 300, 4096, act=1, bias=True, acc=True, seed=5, ldc=300, c_off=0)


@pytest.mark.parametrize("M,N,K", [(32, 300, 4096), (256, 700, 384)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_front_end_epilogue_256mb_context(dev, mode, M, N, K):
    _run(dev, "epilogue 256 MB", "ctx", "s256", mode, M, N, K, act=1, bias=True, acc=True, seed=5 + mode, ldc=N, c_off=0)


@pytest.mark.parametrize("M,N,K", [(512, 3402, 12288), (64, 1984, 8192), (384, 128, 12288)])   # style conv1, speech conv, in_proj
def test_single_pass_weight_gradient_shapes(dev, M, N, K):
    assert M * N * K >= gc.TC_MIN_MACS
    _run(dev, "fast_wgrad", "ctx", "s256fast", 1, M, N, K, seed=M + N + K, ldc=N, c_off=0)


# ---------------------------------------------------------------------------------------------- past 65535 row tiles
@pytest.mark.parametrize("spec,mode,M,N,K", [
    ("m0", 0, 4_194_305, 3, 5),       # SIMT: 65536 tiles of 64 rows
    ("m0", 2, 8_388_481, 3, 5),       # n32 kernel: 65536 tiles of 128 rows
    ("big", 0, 8_388_481, 8, 8),      # tensor cores: 65536 tiles of 128 rows
    ("big", 1, 2, 2, 2_097_153),      # mode 1: the transposing split of A and B over 65538 tiles of 32 contraction rows
])
def test_products_past_the_row_tile_grid_limit(dev, spec, mode, M, N, K):
    _run(dev, "grid limit", "ctx", spec, mode, M, N, K, act=1, bias=True, acc=True, seed=17)
