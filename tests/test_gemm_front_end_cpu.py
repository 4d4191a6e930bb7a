"""CPU-only checks of the GEMM front end's context rules: a zeggs_ctx whose gemm_mode is neither 0 (fp32 SIMT) nor 1 (tensor-core
split-bf16) is refused before anything is launched, so no device is needed to see it."""
import ctypes as C

import pytest

from tests._util import ensure_built


@pytest.fixture(scope="module")
def built():
    ensure_built()
    from zeggs_b200 import _lib
    return _lib


@pytest.mark.parametrize("layout", [0, 1, 2])
def test_gemm_f32_ctx_refuses_an_unknown_gemm_mode(built, layout):
    l = built.lib()
    ctx = built.Ctx(scratch=None, scratch_bytes=0, gemm_mode=2, fast_wgrad=0)
    M, N, K = 256, 384, 512
    rc = l.zeggs_gemm_f32_ctx(C.addressof(ctx), layout, M, N, K, None, K, None, K, None, None, N, 0, 0, None)
    assert rc == -1                                             # ZEGGS_ERR_ARG
    assert b"zeggs_ctx.gemm_mode" in l.zeggs_last_error()


def test_set_gemm_mode_accepts_only_0_and_1(built):
    from zeggs_b200 import ops
    with pytest.raises(built.ZeggsError):
        ops.set_gemm_mode(2)
    assert ops.GEMM_MODE in (0, 1)
