"""numpy restatements of the training-set kernels (csrc/dataset.cu).  zeggs_spline_resample: the chunked not-a-knot cubic spline that stands in for
scipy's griddata(method="cubic") in 1-D.  Same recurrences, same chunking and halo, vectorised over chunks and channels, so the
CPU tests can pin the algorithm against scipy at sizes the GPU sees (tests/test_data_pipeline_cpu.py)."""
import numpy as np

R = 2.0 - np.sqrt(3.0)
G0 = 1.0 / (2.0 * np.sqrt(3.0))
CHUNK, HALO = 256, 48


def linspace_positions(n, m):
    """np.linspace(0, n-1, m) as the kernel computes it: k * ((n-1)/(m-1)), the last exactly n-1."""
    if m <= 1:
        return np.zeros(m)
    x = np.arange(m, dtype=np.float64) * ((n - 1) / (m - 1))
    x[-1] = n - 1
    return x


def second_derivatives(y):
    """y [n, C] -> M [n, C] of the not-a-knot spline on the grid 0..n-1, by the kernel's chunked causal / anticausal recursions."""
    y = np.asarray(y, dtype=np.float64)
    n, C = y.shape
    rhs = np.zeros((n, C))
    if n >= 5:
        rhs[2:n - 2] = 6.0 * ((y[1:n - 3] - 2.0 * y[2:n - 2]) + y[3:n - 1])
    M = np.zeros((n, C))
    n_chunks = (n + CHUNK - 1) // CHUNK
    i0 = np.arange(n_chunks) * CHUNK
    i1 = np.minimum(n, i0 + CHUNK)
    # forward: P runs from max(1, i0 - HALO) to i1 - 1
    start = np.maximum(1, i0 - HALO)
    P = np.zeros((n_chunks, C))
    for s in range(CHUNK + HALO):
        k = start + s
        live = k < i1
        kk = np.minimum(k, n - 1)
        P = np.where(live[:, None], rhs[kk] - R * P, P)
        w = live & (k >= i0)
        M[kk[w]] = G0 * P[w]
    # backward: Q from min(n-2, i1 - 1 + HALO) down to max(1, i0)
    top = np.minimum(n - 2, i1 - 1 + HALO)
    low = np.maximum(1, i0)
    Q = np.zeros((n_chunks, C))
    for s in range(CHUNK + HALO):
        k = top - s
        live = k >= low
        kk = np.maximum(k, 0)
        w = live & (k < i1)
        M[kk[w]] += G0 * Q[w]
        Q = np.where(live[:, None], -R * (rhs[kk] + Q), Q)
    # restore M_1 = d_1 and M_{n-2} = d_{n-2} with the two decaying homogeneous solutions
    d = lambda i: (y[i - 1] - 2.0 * y[i]) + y[i + 1]
    e1, e2 = d(1) - M[1], d(n - 2) - M[n - 2]
    rho = (-R) ** (n - 3) if n - 3 < 64 else 0.0
    det = 1.0 - rho * rho
    alpha, beta = (e1 - rho * e2) / det, (e2 - rho * e1) / det
    i = np.arange(1, n - 1)
    h1 = np.where(i - 1 < 64, (-R) ** np.minimum(i - 1, 64), 0.0)
    h2 = np.where(n - 2 - i < 64, (-R) ** np.minimum(n - 2 - i, 64), 0.0)
    M[1:n - 1] += h1[:, None] * alpha[None] + h2[:, None] * beta[None]
    M[0] = 2.0 * M[1] - M[2]
    M[n - 1] = 2.0 * M[n - 2] - M[n - 3]
    return M


def spline_resample(x, m):
    """x [n] or [n, ...] -> [m] or [m, ...] float64: the spline through x at linspace(0, n-1, m)."""
    x = np.asarray(x)
    n = x.shape[0]
    if n < 4:
        raise ValueError("a cubic spline needs at least 4 samples")
    y = x.reshape(n, -1).astype(np.float64)
    M = second_derivatives(y)
    xs = linspace_positions(n, m)
    i = np.clip(np.floor(xs).astype(np.int64), 0, n - 2)
    t = (xs - i)[:, None]
    u = 1.0 - t
    out = u * y[i] + t * y[i + 1] + ((u * u * u - u) * M[i] + (t * t * t - t) * M[i + 1]) / 6.0
    return out.reshape((m,) + x.shape[1:])


def unroll_by_scan(q):
    """quat.unroll as zeggs_anim_features computes it: per frame the map s -> a s + b (keep, negate, or reset to +1 on an exact zero
    dot of the raw quaternions), composed by a prefix scan.  q [T, J, 4] -> the unrolled sequence."""
    q = np.asarray(q)
    d = np.sum(q[1:] * q[:-1], axis=-1)
    a = np.where(d > 0, 1, np.where(d < 0, -1, 0))
    b = (d == 0).astype(np.int64)
    s = np.ones(q.shape[1], dtype=np.int64)
    signs = [s]
    for t in range(len(d)):
        s = a[t] * s + b[t]
        signs.append(s)
    return q * np.stack(signs)[..., None]
