"""CPU checks of the BVH MOTION-block text kernels (csrc/bvh_text.cu): the scalar token parser and "%f" formatter they run
(csrc/bvh_text.cuh) are compiled as HOST code into a scratch harness (tests/host/bvh_text_host.cu) and compared with Python's float()
bit for bit and '%f' byte for byte; the new entry points are exported with mirrored struct layouts; the host-side line splitting in
front of the device parser matches Python's universal-newline read.  No GPU involved."""
import ctypes as C
import math
import os
import re
import subprocess
import struct
from fractions import Fraction

import numpy as np
import pytest

from tests._util import ROOT, ensure_built

STRIDE = 48


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("host") / "libzeggs_bvh_text_host.so")     # private directory: no clash with another user's build
    src = os.path.join(ROOT, "tests", "host", "bvh_text_host.cu")
    r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared",
                        "-o", out, src], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip("nvcc host harness build failed: " + r.stderr[-400:])
    return C.CDLL(out)


def P(a):
    return a.ctypes.data_as(C.c_void_p)


def parse(harness, tokens):
    text = "".join(tokens).encode("ascii")
    ends = np.cumsum([len(t) for t in tokens]).astype(np.int64)
    bounds = np.stack([ends - [len(t) for t in tokens], ends], axis=1).astype(np.int64)
    buf = np.frombuffer(text + b"\0", dtype=np.uint8).copy()
    out, ok = np.zeros(len(tokens)), np.zeros(len(tokens), np.int32)
    harness.parse_tokens_host(P(buf), P(bounds), len(tokens), P(out), P(ok))
    return out, ok.astype(bool)


def fmt(harness, values):
    v = np.ascontiguousarray(values, dtype=np.float64)
    out, ln = np.zeros(len(v) * STRIDE, np.uint8), np.zeros(len(v), np.int32)
    harness.format_values_host(P(v), len(v), P(out), STRIDE, P(ln))
    text = out.tobytes()
    return [text[i * STRIDE:i * STRIDE + n].decode("ascii") if n >= 0 else None for i, n in enumerate(ln)], ln


_FAST = re.compile(r"[+-]?(?:(\d+)(?:\.(\d*))?|\.(\d+))(?:[eE]([+-]?\d+))?")


def on_fast_path(tok):
    """The kernel's rule: the grammar, significant digits as an integer <= 2^53, decimal exponent in [-22, 22]."""
    m = _FAST.fullmatch(tok)
    if not m:
        return False
    ip, fp, only = m.group(1), m.group(2), m.group(3)
    digits = (ip + (fp or "")) if ip is not None else only
    k = -len(fp or "") if ip is not None else -len(only)
    k += int(m.group(4) or 0)
    return int(digits) <= 2 ** 53 and -22 <= k <= 22


def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def check_parse(harness, tokens):
    out, ok = parse(harness, tokens)
    for t, v, o in zip(tokens, out, ok):
        assert o == on_fast_path(t), t
        if o:
            assert bits(v) == bits(float(t)), (t, v, float(t))


def test_parse_random_printf_strings_bit_for_bit(harness):
    rs = np.random.RandomState(0)
    mags = 10.0 ** rs.uniform(-7, 6, 20000)
    vals = mags * rs.choice([-1.0, 1.0], mags.size)
    toks = ["%f" % v for v in vals] + ["%.6f" % v for v in vals] + ["%.9g" % v for v in vals]
    toks += ["%f" % np.float32(v) for v in vals[:5000]]
    _, ok = parse(harness, toks)
    assert ok.all()                                  # every printf-made token of these magnitudes is on the fast path
    check_parse(harness, toks)


def test_parse_signs_zeros_points_and_leading_zeros(harness):
    check_parse(harness, ["+1.5", "-1.5", "-0.000000", "0.000000", "+0.0", "-0", ".5", "-.5", "+.5", "5.", "-5.", "007.250",
                          "000000000000000000000000000001.5", "0.0000001", "1E5", "1e+05", "-2.5e-3", "5.e2", ".5E-1"])
    out, ok = parse(harness, ["-0.000000"])
    assert ok[0] and math.copysign(1.0, out[0]) == -1.0


def test_parse_exponent_edges(harness):
    toks = ["1e22", "1e-22", "1e23", "1e-23", "9e22", "1.5e21", "15e21", "0.1e23", "10e-23", "1e-24", "0e30", "123456789e-22"]
    check_parse(harness, toks)
    _, ok = parse(harness, ["1e22", "1e-22", "1e23", "1e-23", "15e21", "10e-23"])
    assert ok.tolist() == [True, True, False, False, True, False]          # 10e-23: s = 10, k = -23


def test_parse_long_significands(harness):
    rs = np.random.RandomState(1)
    toks = []
    for nd in (15, 16, 20):
        for _ in range(300):
            d = "".join(str(x) for x in rs.randint(0, 10, nd))
            d = str(rs.randint(1, 10)) + d[1:]
            cut = rs.randint(0, nd + 1)
            toks.append(("-" if rs.rand() < 0.5 else "") + d[:cut] + "." + d[cut:])
    toks += ["9007199254740992", "9007199254740993", "900719925474099.2", "900719925474099.3", "12345678901234567890"]
    check_parse(harness, toks)
    _, ok = parse(harness, ["9007199254740992", "9007199254740993", "12345678901234567890"])
    assert ok.tolist() == [True, False, False]


def test_tokens_off_the_fast_path_are_flagged(harness):
    toks = ["nan", "NaN", "-nan", "inf", "-inf", "Infinity", "1_000", "1.2.3", "abc", "+", "-", ".", "e5", "1e", "1e+", "0x10",
            "--1", "1.5f", "1,5", "1e99999999", "1" * 40, "0." + "0" * 30 + "1", "1\x00", "\x7f"]
    _, ok = parse(harness, toks)
    assert not ok.any(), [t for t, o in zip(toks, ok) if o]


def test_format_random_float32_and_float64_byte_for_byte(harness):
    rs = np.random.RandomState(2)
    n = 500_000
    mags = 10.0 ** rs.uniform(-9, 9, n) * rs.choice([-1.0, 1.0], n)
    f64 = np.concatenate([mags[: n // 2], rs.randn(n // 2) * 180.0])
    f32 = np.concatenate([mags[n // 2:].astype(np.float32), (rs.randn(n // 2) * 180.0).astype(np.float32)]).astype(np.float64)
    for v in (f64, f32):
        got, ln = fmt(harness, v)
        assert (ln >= 0).all()
        want = ["%f" % x for x in v.tolist()]
        bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
        assert not bad, [(v[i], got[i], want[i]) for i in bad[:5]]


def test_format_ties_signs_and_specials(harness):
    vals = [1 / 128, 3 / 128, 5 / 128, -1 / 128, 0.5e-6, 1.5e-6, 2.5e-6, -2.5e-6, 0.0000005, 2 ** -21, 3 * 2 ** -21, 1e-7, -1e-7,
            0.0, -0.0, -1e-300, -5e-324, 5e-324, 1e-320, float("nan"), -float("nan"), float("inf"), -float("inf"),
            2.0 ** 53, 2.0 ** 53 + 2, 2.0 ** 64, 1e20, -1e25, 0.1, 0.7, 123.4567895]
    vals += [k / 2 ** 7 for k in range(-300, 300)] + [k / 2 ** 21 for k in range(0, 4000, 7)]
    got, ln = fmt(harness, vals)
    assert got[:2] == ["0.007812", "0.023438"]
    assert got[got.index("-0.000000")] == "-0.000000" and ("%f" % -0.0) == "-0.000000"
    assert [g for g in got] == ["%f" % x for x in vals]


def test_format_largest_value_of_the_128_bit_path(harness):
    limit = Fraction(2 ** 128, 10 ** 6)
    x = float(limit)
    while Fraction(x) >= limit:
        x = math.nextafter(x, 0.0)
    while Fraction(math.nextafter(x, math.inf)) < limit:
        x = math.nextafter(x, math.inf)
    beyond = math.nextafter(x, math.inf)
    got, ln = fmt(harness, [x, -x, beyond, -beyond, 1e300, -1e308])
    assert got[0] == "%f" % x and got[1] == "%f" % -x and len(got[1]) <= 41
    assert ln[2:].tolist() == [-1, -1, -1, -1]


# ---------------------------------------------------------------------------------------------- ABI
NEW = ("zeggs_bvh_parse_motion_workspace_size", "zeggs_bvh_parse_motion", "zeggs_bvh_format_motion_max_size",
       "zeggs_bvh_format_motion_workspace_size", "zeggs_bvh_format_motion")


@pytest.fixture(scope="module")
def built():
    ensure_built()
    from zeggs_b200 import _lib
    return _lib


def test_bvh_entry_points_are_exported_and_mirrored(built):
    l = built.lib()
    bound = {s[0] for s in built.SYMBOLS}
    hdr = open(os.path.join(ROOT, "include", "zeggs_b200.h")).read()
    for name in NEW:
        assert name in bound and re.search(r"\b%s\s*\(" % name, hdr) and getattr(l, name) is not None
    mirrors = built.struct_mirrors()
    for name in ("zeggs_bvh_parse_args", "zeggs_bvh_format_args"):
        assert l.zeggs_struct_size(name.encode()) == C.sizeof(mirrors[name]) > 0, name


def test_bvh_sizes_and_argument_checks(built):
    l = built.lib()
    assert l.zeggs_bvh_format_motion_max_size(3600, 75) == 3600 * 228 * 42 + 3600
    assert l.zeggs_bvh_format_motion_max_size(0, 75) == 0 and l.zeggs_bvh_format_motion_max_size(1, 0) == 0
    assert l.zeggs_bvh_parse_motion_workspace_size(20_000_000, 9000) >= 4 * 20_000_000 + 4 * 9000
    assert l.zeggs_bvh_parse_motion_workspace_size(1 << 31, 10) == 0 and l.zeggs_bvh_parse_motion_workspace_size(-1, 10) == 0
    assert l.zeggs_bvh_format_motion_workspace_size(3600, 75) > 0
    dummy = C.create_string_buffer(64)
    p = C.addressof(dummy)
    launches = l.zeggs_launch_count()
    a = built.BvhParseArgs(n_bytes=100, n_frames=2, C=6, max_flagged=4, text=p, out=p, flagged=p, status=p, workspace=p, workspace_bytes=8)
    assert l.zeggs_bvh_parse_motion(C.byref(a), None) != 0 and "workspace" in l.zeggs_last_error().decode()
    f = built.BvhFormatArgs(T=2, J=2, in_f64=0, positions=p, rotations=p, seq=p, out=p, out_capacity=10, row_start=p, status=p,
                            workspace=p, workspace_bytes=1 << 20)
    assert l.zeggs_bvh_format_motion(C.byref(f), None) != 0 and "needed" in l.zeggs_last_error().decode()
    assert l.zeggs_launch_count() == launches


# ---------------------------------------------------------------------------------------------- host side of the device parser
@pytest.mark.parametrize("nl", ["\n", "\r\n", "\r"])
def test_header_split_matches_universal_newline_read(tmp_path, nl):
    from tests import _fixtures as fx
    from zeggs_b200 import animation
    src = fx.make_synthetic_bvh(str(tmp_path / "s.bvh"), frames=5)
    text = open(src).read().replace("\n", nl)
    p = tmp_path / "n.bvh"
    p.write_bytes(text.encode("ascii"))
    with open(p, "r") as f:
        lines = iter(f.read().split("\n"))
    want = animation._parse_header(lines)
    want_rows = [r for r in lines if r.strip()]
    raw = p.read_bytes()
    state = {}
    got = animation._parse_header(animation._header_lines(memoryview(raw), state))
    assert got == want
    rest = raw[state["next"]:].decode("ascii").replace("\r\n", "\n").replace("\r", "\n")
    assert [r for r in rest.split("\n") if r.strip()] == want_rows
