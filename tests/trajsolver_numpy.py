"""The TrajSolver closed form restated with numpy's LAPACK-backed dense algebra, shared by the tests that bound the oracle's
(and so the GPU's) rounding against an implementation that shares no code with it."""
import math

import numpy as np


def numpy_poly_solve(dim, N, R, wps, dts, ncol_get):
    """The same closed form with numpy's LAPACK-backed dense algebra (an implementation that shares no code with the oracle or
    the stand-in Eigen): assembles A, Q, M exactly as poly_solver.cpp:40-171 does and solves with np.linalg.solve."""
    W, S, H = len(wps), len(wps) - 1, N // 2
    A = np.zeros((S * N, S * N))
    Q = np.zeros((S * N, S * N))
    for i in range(S):
        T = dts[i]
        for n in range(N):
            if n < H:
                A[i * N + n, i * N + n] = math.factorial(n)
            for r in range(H):
                if r <= n:
                    A[i * N + H + r, i * N + n] = math.factorial(n) // math.factorial(n - r) * T ** (n - r)
            for r in range(N):
                if r >= R and n >= R:
                    val = 1
                    for m in range(R):
                        val *= (r - m) * (n - m)
                    Q[i * N + r, i * N + n] = val * T ** (r + n - 2 * R + 1) / (r + n - 2 * R + 1)
    use = lambda w, k: (int(w["control"]) >> k) & 1  # noqa: E731
    nfixed = sum(use(w, k) for w in wps for k in range(H))
    table, raw, fix, fre = [], 0, 0, 0
    for wid, w in enumerate(wps):
        interior = 0 < wid < W - 1
        for k in range(H):
            nid = fix if use(w, k) else nfixed + fre
            table.append((raw, nid, wid, k))
            if interior:
                table.append((raw + H, nid, wid, k))
            raw += 1
            if use(w, k):
                fix += 1
            else:
                fre += 1
        if interior:
            raw += H
    M = np.zeros((S * N, W * H))
    for r, nid, _, _ in table:
        M[r, nid] = 1
    X = np.linalg.solve(A, M)
    Rm = X.T @ Q @ X
    D = np.zeros((W * H, dim))
    for r, nid, wid, k in table:
        if nid < nfixed:
            D[nid] = ncol_get(wps[wid], k)
    nfree = W * H - nfixed
    if W > 2 and nfree > 0:
        D[nfixed:] = -np.linalg.solve(Rm[nfixed:, nfixed:], Rm[nfixed:, :nfixed] @ D[:nfixed])
    d = M @ D
    out = np.zeros((S, dim, 6))
    for i in range(S):
        p = np.linalg.solve(A[i * N:(i + 1) * N, i * N:(i + 1) * N], d[i * N:(i + 1) * N])
        for a in range(dim):
            c = np.zeros(6)
            for k in range(N):
                c[k] = p[k, a] * math.factorial(k)
            out[i, a] = c[::-1]
    return out
