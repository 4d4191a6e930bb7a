"""GPU: the loudness meter (csrc/loudness.cu, zeggs_loudness_gain) through LoudnessMeter.gain(..., want_lufs=True) against
oracle/loudness_oracle.py (pyloudnorm 0.1.0 restated in float64) at every shape and edge it accepts.

* Bounds: where the oracle's loudness is finite, |L - L_ref| <= 1e-5 LU and |g - g_ref| <= 2e-6 g_ref; where nothing passes the
  absolute gate (all-zero clips, a constant 1e-5, noise near -80 LUFS), L = -inf and g = +inf exactly.
* Lengths at 16 kHz: one sample short of a block (refused), one block, around the rounding of the block count at 8000 samples,
  a ragged and a clamped last block, 10 s and 1 minute; 5952, 5953, 6000 and 6001 blocks (about ten minutes) and 20 minutes.
* Rates 8000, 11025 (uneven segments), 22050, 44100 and 48000 Hz, each with a meter of its own.
* Content: speech-like, white noise, 38 Hz on a DC offset, 1.5 kHz, a clipped square, a burst in near-silence, sections that put
  the relative threshold below -70 LUFS, silence and sub-gate clips.  Batches of 1, 3, 128, 129 and 300, float32 and int16.
* Bitwise: each clip of a batch equals the clip alone; int16 equals float32 x / 32768; a repeated call is identical; one meter
  at two lengths in turn equals two fresh meters.
tests/test_loudness_f64_cpu.py shows a restatement of the kernel's scheme meets these bounds with >= 4x headroom and that each
modelled fault breaks one.
"""
import numpy as np
import pytest
import torch

from tests import _loudness_cases as lc
from tests._util import ensure_built

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    ensure_built()
    return torch.device("cuda:0")


def _meter(dev, rate=16000):
    from zeggs_b200 import audio
    return audio.LoudnessMeter(dev, rate)


def _run(meter, x):
    gain, lufs = meter.gain(torch.from_numpy(np.ascontiguousarray(x)).to(meter.device), want_lufs=True)
    return gain.cpu().numpy(), lufs.cpu().numpy()


def _check(tag, meter, x, rate):
    """One call on x [N, n]; every clip against the oracle.  -> worst ratio, printed with its clip."""
    gain, lufs = _run(meter, x)
    worst, at = -1.0, None
    for i in range(x.shape[0]):
        L, g = lc.oracle(x[i], rate)
        r = lc.ratio(lufs[i], gain[i], L, g)
        if not r <= worst:
            worst, at = r, (i, L, float(lufs[i]))
    print(f"  [{tag}] worst {worst:.3g} of the bound (clip {at[0]}: {at[2]!r} vs oracle {at[1]!r} LUFS)")
    assert worst <= 1.0, tag
    return gain, lufs


# ---------------------------------------------------------------------------------------------- lengths
def test_shorter_than_one_block_is_refused(dev):
    from zeggs_b200 import _lib
    with pytest.raises(_lib.ZeggsError):
        _meter(dev).gain(torch.zeros(2, lc.TOO_SHORT, device=dev))


@pytest.mark.parametrize("n", lc.LEN_16K)
def test_lengths_at_16k_every_content(dev, n):
    x = np.stack([lc.content(k, n, 16000, 7) for k in lc.CONTENTS])
    _check(f"16 kHz n{n}", _meter(dev), x, 16000)


@pytest.mark.parametrize("blocks", lc.BLOCK_COUNTS + ["20min"])
def test_long_clips(dev, blocks):
    """About ten minutes, across 48 KB of per-block doubles and the former 6000-block cap, and 20 minutes: metered like any
    other clip.  Two clips per call: speech-like and the gate sections."""
    n = lc.MIN_20 if blocks == "20min" else lc.samples_for_blocks(blocks)
    x = np.stack([lc.content("speech", n, 16000, 1), lc.content("gate_sections", n, 16000, 2)])
    _check(f"{blocks} blocks, n{n}", _meter(dev), x, 16000)


@pytest.mark.parametrize("rate", lc.OTHER_RATES)
def test_other_rates(dev, rate):
    m = _meter(dev, rate)
    for n in lc.rate_lengths(rate):
        x = np.stack([lc.content(k, n, rate, 11) for k in lc.CONTENTS])
        _check(f"{rate} Hz n{n}", m, x, rate)


# ---------------------------------------------------------------------------------------------- batches and invariances
@pytest.mark.parametrize("n_clips", [1, 3, 128, 129, 300])
def test_batches_float32_and_int16(dev, n_clips):
    """One call per batch against the oracle, then bitwise: each clip alone, the int16 batch against float32 x / 32768, and a
    repeated call."""
    n = lc.clamped_length(16000)
    x = lc.batch(n_clips, n, 16000, seed=n_clips)
    m = _meter(dev)
    gain, lufs = _check(f"{n_clips} clips float32", m, x, 16000)
    x16 = lc.to_pcm16(x)
    gain16, lufs16 = _check(f"{n_clips} clips int16", m, x16, 16000)
    g2, l2 = _run(m, x)
    assert np.array_equal(g2.view(np.uint32), gain.view(np.uint32)) and np.array_equal(l2.view(np.uint32), lufs.view(np.uint32))
    gd, ld = _run(m, (x16.astype(np.float32) / np.float32(32768.0)))
    assert np.array_equal(gd.view(np.uint32), gain16.view(np.uint32)) and np.array_equal(ld.view(np.uint32), lufs16.view(np.uint32))
    alone = [_run(m, x[i:i + 1]) for i in range(n_clips)]
    ga = np.concatenate([a[0] for a in alone])
    la = np.concatenate([a[1] for a in alone])
    assert np.array_equal(ga.view(np.uint32), gain.view(np.uint32)) and np.array_equal(la.view(np.uint32), lufs.view(np.uint32))


def test_one_meter_at_two_lengths_equals_fresh_meters(dev):
    """The geometry cache: one meter called at 160000, 48900 and 160000 samples gives the bits of a fresh meter at each."""
    a = lc.batch(4, 160000, 16000, seed=3)
    b = lc.batch(4, lc.clamped_length(16000), 16000, seed=4)
    m = _meter(dev)
    seq = [_run(m, a), _run(m, b), _run(m, a)]
    fresh = [_run(_meter(dev), a), _run(_meter(dev), b)]
    for got, ref in zip(seq, [fresh[0], fresh[1], fresh[0]]):
        for u, v in zip(got, ref):
            assert np.array_equal(u.view(np.uint32), v.view(np.uint32))
