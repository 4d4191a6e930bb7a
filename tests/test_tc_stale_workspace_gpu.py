"""GPU: the tensor-core decoder's results do not depend on what its training workspace held before the call.

A training forward takes a fresh workspace from PyTorch's caching allocator, and the grow-only workspaces of the backward are
allocated afresh whenever a call needs more, so they start with whatever an earlier, freed tensor left there.  Batch-padding lanes
(b >= B inside the 32-sample tile) go through the weight-gradient products with zero gradients, and a stale NaN in one of their
history columns would turn those zeros into NaN.  Here the allocator's only free segment is filled with
0xFF bytes (a NaN in every float) before the window, and every output and gradient must be finite and bitwise equal to the same
window run on a zero-filled segment."""
import pytest
import torch

from tests.test_tc_engine_gpu import _case, _run_gpu, dev, engine  # noqa: F401

pytestmark = pytest.mark.gpu


def _on_stale_memory(dev, fill, run):
    from zeggs_b200 import ops
    torch.cuda.synchronize()
    ops.WS.bufs.clear()             # the grow-only workspaces and the GEMM scratch are allocated afresh, from the filled segment too
    ops._scratch.clear()
    torch.cuda.empty_cache()
    seg = torch.full((512 << 20,), fill, dtype=torch.uint8, device=dev)   # every later large allocation is carved from this segment
    del seg
    return run()


@pytest.mark.parametrize("H,B,T", [(384, 16, 12), (512, 1, 5)])
def test_tc_window_ignores_stale_workspace_contents(dev, engine, H, B, T):
    engine("tc")
    case = _case(H, B, T, 64, seed=4100 + H + B + T)
    run = lambda: _run_gpu(dev, *case, H, 64, grads=True)
    out0, g0 = _on_stale_memory(dev, 0, run)
    out1, g1 = _on_stale_memory(dev, 0xFF, run)
    for a, b in zip(out0, out1):
        assert bool(torch.isfinite(b).all()) and torch.equal(a, b)
    bad = [k for k in g0 if not (bool(torch.isfinite(g1[k]).all()) and torch.equal(g0[k], g1[k]))]
    assert not bad, bad
