"""The counter-based draws of csrc/radam.cu restated in numpy: the dropout masks of zeggs_dropout_mask and zeggs_dropout_mask_dev
and the normals of zeggs_randn_dev (the VAE noise).  Every value is defined per element index from (seed, index), so it does not
depend on the launch shape.

* `mix_u32(seed, i)`: the splitmix64 finaliser of seed + golden * (i + 1), top 32 bits.  uint64 arithmetic wraps like the kernel's.
* `device_seed(t, salt)`: the effective seed the device-seeded kernels hash from the seed word t and the salt.
* Masks: thr = (uint32) min(4294967040f, p * 2^32) in float32, keep_scale = 1.0f / (1.0f - p) in float32; mask = keep_scale where
  u32 >= thr, else 0.  Bit-exact.
* Normals: Box-Muller on the words of indices 2k and 2k + 1.  u1 = (float(u32) + 1.0f) * 2^-32 and the angle 6.2831855f * u2 are
  formed exactly in float32 as the kernel forms them; log, sqrt, cos and sin are then evaluated in float64.  The kernel's logf,
  sqrtf and sincosf are within a few fp32 ulps of that.  Since u1 >= 2^-32, |x| <= sqrt(-2 ln 2^-32) = sqrt(64 ln 2) = 6.66: the
  draws have no tail beyond 6.66 sigma (torch.randn has one; P(|x| > 6.66) = 2.7e-11 for a true normal).
"""
import numpy as np

M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15
C1, C2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
SEED_MUL = 0xD1342543DE82EF95
TAIL = float(np.sqrt(64.0 * np.log(2.0)))           # the largest |x| the normals can take


def _finalise(z):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(C1)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(C2)
    return z ^ (z >> np.uint64(31))


def mix_u32(seed, idx):
    """uint32 word of every index in idx (uint64 array-like) under the 64-bit seed."""
    i = np.asarray(idx, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + np.uint64(GOLDEN) * (i + np.uint64(1))
        return (_finalise(z) >> np.uint64(32)).astype(np.uint32)


def device_seed(t, salt):
    """The effective seed of the device-seeded kernels: hash of the seed word t and salt."""
    with np.errstate(over="ignore"):
        z = np.array([t], dtype=np.uint64) * np.uint64(SEED_MUL) + (np.uint64(salt) + np.uint64(1)) * np.uint64(GOLDEN)
        return int(_finalise(z)[0])


def words(n, seed):
    return mix_u32(seed, np.arange(n, dtype=np.uint64))


def threshold(p):
    """(uint32) fminf(4294967040.0f, p * 4294967296.0f), all in float32: P(u32 < thr) = p."""
    t = np.minimum(np.float32(4294967040.0), np.float32(p) * np.float32(4294967296.0))
    return int(t)


def keep_scale(p):
    return np.float32(1.0) / (np.float32(1.0) - np.float32(p))


def mask_from_words(u, p):
    return np.where(u >= np.uint32(threshold(p)), keep_scale(p), np.float32(0.0)).astype(np.float32)


def dropout_mask(n, p, seed):
    """zeggs_dropout_mask(out, n, p, seed): float32 [n]."""
    return mask_from_words(words(n, seed), p)


def dropout_mask_dev(n, p, t, salt):
    """zeggs_dropout_mask_dev with *seed_dev = t: float32 [n]."""
    return mask_from_words(words(n, device_seed(t, salt)), p)


def box_muller_inputs(n, seed):
    """-> (u1, angle) float32 [ceil(n / 2)], exactly as the kernel forms them from the words of indices 2k and 2k + 1."""
    k = np.arange((n + 1) // 2, dtype=np.uint64)
    a = mix_u32(seed, 2 * k).astype(np.float32)                   # round to nearest, as (float) of a uint32
    b = mix_u32(seed, 2 * k + 1).astype(np.float32)
    inv = np.float32(1.0 / 4294967296.0)
    u1 = (a + np.float32(1.0)) * inv                                 # (0, 1]
    ang = np.float32(6.283185307179586) * (b * inv)
    return u1, ang


def randn_dev(n, t, salt):
    """zeggs_randn_dev with *seed_dev = t, in float64 from the kernel's float32 u1 and angle: [n]."""
    u1, ang = box_muller_inputs(n, device_seed(t, salt))
    r = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    out = np.empty(2 * len(u1))
    out[0::2] = r * np.cos(ang.astype(np.float64))
    out[1::2] = r * np.sin(ang.astype(np.float64))
    return out[:n]


# ---------------------------------------------------------------------------------------------- plain-int second implementation
def mix_u32_int(seed, i):
    """mix_u32 in Python ints masked to 64 bits: an independent statement of the same generator."""
    z = (seed + GOLDEN * (i + 1)) & M64
    z = ((z ^ (z >> 30)) * C1) & M64
    z = ((z ^ (z >> 27)) * C2) & M64
    return (z ^ (z >> 31)) >> 32


def device_seed_int(t, salt):
    z = (t * SEED_MUL + (salt + 1) * GOLDEN) & M64
    z = ((z ^ (z >> 30)) * C1) & M64
    z = ((z ^ (z >> 27)) * C2) & M64
    return z ^ (z >> 31)
