"""TensorBoard logs of train() on the GPU: LossLog brings every step's loss terms to the host bitwise (graph replay and eager launches,
lanes on and off) without a sync on the pushes that do not close a block; train() with use_tensorboard writes every optimizer step
exactly once, across a resume too, plus the held-out loss, without changing the training trajectory; under data parallelism the
logged rows are the mean over the ranks and the step keeps its one gradient all-reduce."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests._util import ROOT
from tests.test_dp_nccl_gpu import _free_port
from tests.test_tensorboard_cpu import hparams_of, loss_series
from tests.test_validation_cpu import make_files
from tests.test_validation_gpu import _batch, _final_params, _make_step, _options, decoder_engine, dev  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _collect(step, log, batches, record):
    """One step per batch, each followed by log.push; the terms each step left, cloned on the test's side, go to `record`.
    -> (what every push returned, what the final drain returned), as (steps, rows) pairs."""
    pushed = []
    for b in batches:
        step.step(b)
        record.append(step.terms.clone())
        pushed.append(log.push(step))
    return pushed, log.drain()


@pytest.mark.parametrize("lanes", ["1", "0"])
@pytest.mark.parametrize("use_graph", [True, False])
def test_collector_rows_equal_the_step_terms(dev, decoder_engine, monkeypatch, use_graph, lanes):
    """10 steps in blocks of 4 (the last one partial): the rows equal the terms of their steps bitwise, at steps 0..9; a push
    returns rows only when it closes a block, and then the previous block's."""
    from zeggs_b200.train import LossLog
    decoder_engine("fp32")
    monkeypatch.setenv("ZEGGS_LANES", lanes)
    torch.manual_seed(3)
    step, _ = _make_step(dev, 64, "example", seed=8, use_graph=use_graph)
    assert step.lanes == (lanes == "1")
    log = LossLog(dev, block=4)
    rec = []
    pushed, (ds, dr) = _collect(step, log, [_batch(dev, 4, 16, 24, 70 + i) for i in range(10)], rec)
    torch.cuda.synchronize()
    if use_graph:
        assert step.use_graph and len(step._graphs) == 1, "the CUDA-graph path did not run"
    assert [len(s) for s, _ in pushed] == [0, 0, 0, 0, 0, 0, 0, 4, 0, 0]
    steps = np.concatenate([s for s, _ in pushed] + [ds])
    rows = np.concatenate([r for _, r in pushed] + [dr])
    assert steps.tolist() == list(range(10))
    want = torch.stack(rec).cpu().numpy()
    assert len(np.unique(want[:, 0])) == 10                  # every step left different terms
    assert rows.dtype == np.float32 and rows.tobytes() == want.tobytes()
    assert log.drain()[0].size == 0


def test_pushes_inside_a_block_do_not_sync(dev, decoder_engine):
    """Three blocks of graph-replayed steps with sync debug mode "error" around every push that does not close its block."""
    from zeggs_b200.train import LossLog
    decoder_engine("fp32")
    torch.manual_seed(4)
    step, _ = _make_step(dev, 64, "example", seed=9, use_graph=True)
    b = _batch(dev, 4, 16, 24, 80)
    for _ in range(2):                                        # eager first sight of the geometry, then the capture
        step.step(b)
    log = LossLog(dev, block=4)
    got = []
    for i in range(12):
        step.step(b)
        closes = i % 4 == 3
        prev = torch.cuda.get_sync_debug_mode()
        if not closes:
            torch.cuda.set_sync_debug_mode("error")
        try:
            s, _ = log.push(step)
        finally:
            torch.cuda.set_sync_debug_mode(prev)
        got += s.tolist()
    got += log.drain()[0].tolist()
    assert len(step._graphs) == 1
    assert got == list(range(2, 14))


# ---------------------------------------------------------------------------------------------- train() end to end
def _run(base, ddef, dproc, gss, n, tb, resume=False):
    from zeggs_b200.train import train
    models, logs = os.path.join(base, "models"), os.path.join(base, "logs")
    to, no = _options(21, gss, n)
    to.update(use_tensorboard=tb, resume=resume)
    state = random.getstate()
    random.seed(0)
    try:
        train(models, logs, dproc, ddef, to, no)
    finally:
        random.setstate(state)
    return models, logs


def _assert_every_step_once(tb_dir, n):
    ser = loss_series(tb_dir)
    for name, pts in ser.items():
        assert sorted(s for s, _ in pts) == list(range(n)), name
    return ser


def test_train_writes_every_step_and_keeps_the_trajectory(dev, tmp_path, decoder_engine):
    ddef, dproc = make_files(str(tmp_path / "data"))
    n, gss = 250, 125
    models, logs = _run(str(tmp_path / "a"), ddef, dproc, gss, n, True)
    tb_dir = os.path.join(logs, "tb")
    ser = _assert_every_step_once(tb_dir, n)
    terms = np.array([[v for _, v in sorted(ser[k])] for k in ser], dtype=np.float64).T        # [n, 19]
    assert np.all(np.isfinite(terms))
    err = np.abs(terms[:, 0] - terms[:, 1:].sum(1) / 18)
    assert np.all(err <= 2e-6 * np.abs(terms[:, 1:]).sum(1) / 18), err.max()
    assert hparams_of(tb_dir)["decoder_nhidden"] == 64
    recs = [json.loads(ln) for ln in open(os.path.join(logs, "valid_loss.jsonl")).read().strip().split("\n")]
    assert [r["iteration"] for r in recs] == [125, 250]
    val = loss_series(tb_dir, "valid")
    for name in val:
        assert [(s, np.float32(v)) for s, v in val[name]] == [(r["iteration"], np.float32(r["valid"][name])) for r in recs], name
    # the logging does not touch the training trajectory
    models_b, logs_b = _run(str(tmp_path / "b"), ddef, dproc, gss, n, False)
    assert not os.path.exists(os.path.join(logs_b, "tb"))
    pa, pb = _final_params(models), _final_params(models_b)
    assert set(pa) == set(pb)
    for k in pa:
        assert torch.equal(pa[k], pb[k]), k


def test_resumed_run_continues_the_steps(dev, tmp_path, decoder_engine):
    """A run that ends at its checkpoint (iteration 120) and a resumed run into the same directories to 250: every step once over
    the event files of both."""
    ddef, dproc = make_files(str(tmp_path / "data"))
    base = str(tmp_path / "run")
    _run(base, ddef, dproc, 60, 120, True)
    _, logs = _run(base, ddef, dproc, 60, 250, True, resume=True)
    tb_dir = os.path.join(logs, "tb")
    _assert_every_step_once(tb_dir, 250)
    assert [s for s, _ in loss_series(tb_dir, "valid")["total"]] == [60, 120, 180, 240]


def test_data_parallel_rows_are_rank_means():
    """2 ranks (NCCL): rank 0's collected rows equal (t0 + t1) * 0.5 of the ranks' per-step terms in fp32, and every step makes
    exactly one gradient all-reduce."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "tb_dp_worker.py")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("TBDPRESULT ")][-1]
    d = json.loads(line[len("TBDPRESULT "):])
    print(" ", d)
    assert d["steps"] == list(range(10))
    assert d["graphed"] and d["rows_equal_rank_mean"] and d["ranks_differ"]
    assert d["allreduces"] == 10
