"""CPU restatement of the local-loop-closure deformation solve (test infrastructure only).

Deformation::constrain with fernMatch = relaxGraph = false (reference Core/Deformation.cpp:73-207) on top of
DeformationGraph (Core/Utils/DeformationGraph.cpp): constraint weighting (weightVerticesSeq, :268-373), the Jacobian and
residual rows exactly as sparseJacobian / sparseResidual build them (:494-887), and at most three Gauss-Newton iterations
(optimiseGraphSparse, :416-492). The reference solves JᵀJ δ = -Jᵀr with CHOLMOD under a fill-reducing permutation; this
restatement materialises J as a sparse matrix, forms JᵀJ with scipy and factorises it with LAPACK's band Cholesky in time
order, so it shares no arithmetic with the device solver (ef_deform.cu), which assembles the normal equations directly.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

K = 4            # DeformationGraph::k (Deformation.cpp:23)
LOOKBACK = 20
W_REG, W_CON = 10.0, 100.0
NV = 12


def neighbours(n, k=K):
    """connectGraphSeq (:239-266)."""
    out = [[] for _ in range(n)]
    for i in range(k // 2):
        out[i] = [m for m in range(k + 1) if m != i]
    for i in range(k // 2, n - k // 2):
        for m in range(k // 2):
            out[i] += [i - (m + 1), i + (m + 1)]
    for i in range(n - k // 2, n):
        out[i] = [m for m in range(n - (k + 1), n) if m != i]
    return out


def _norm(v):
    return np.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])


def weight_point(pos, times, p, t):
    """weightVerticesSeq for one point: (k node ids ascending, their normalised weights)."""
    n = len(times)
    imin, imax = 0, n - 1
    imid = (imin + imax) // 2
    while imax >= imin:
        imid = (imin + imax) // 2
        if times[imid] < t:
            imin = imid + 1
        elif times[imid] > t:
            imax = imid - 1
        else:
            break
    imin = min(imin, n - 1)
    di, dm = abs(int(times[imin]) - t), abs(int(times[imid]) - t)
    dx = abs(int(times[imax]) - t) if imax >= 0 else None  # imax < 0: every choice gives the window 0..19
    if di <= dm and (dx is None or di <= dx):
        found = imin
    elif dm <= di and (dx is None or dm <= dx):
        found = imid
    else:
        found = max(imax, 0)
    win = list(range(found, max(found - LOOKBACK, -1), -1))
    win += list(range(found + 1, n))[:LOOKBACK - len(win)]
    dist = [np.float32(_norm(pos[j] - p)) for j in win]
    order = sorted(range(len(win)), key=lambda i: dist[i])  # stable
    dmax = float(dist[order[K]])
    ids = [win[i] for i in order[:K]]
    w = [(1.0 - _norm(p - pos[j]) / dmax) ** 2 for j in ids]
    s = 0.0
    for x in w:
        s += x
    w = [x / s for x in w]
    o = sorted(range(K), key=lambda i: ids[i])
    return [ids[i] for i in o], [w[i] for i in o]


def expand_constraints(src, dst, src_times, dst_times, pin):
    """Deformation::addConstraint (:73-86): [c0, pin0, c1, pin1, ...] with pins (target, target, t, t)."""
    S, D, T = [], [], []
    for i in range(len(src)):
        S.append(np.asarray(src[i], np.float64)); D.append(np.asarray(dst[i], np.float64)); T.append(int(src_times[i]))
        if pin:
            S.append(np.asarray(dst[i], np.float64)); D.append(np.asarray(dst[i], np.float64)); T.append(int(dst_times[i]))
    return np.array(S).reshape(-1, 3), np.array(D).reshape(-1, 3), np.array(T, np.int64)


class Solver:
    def __init__(self, pos, times, src, dst, ctimes, last_deform_time):
        self.pos = np.asarray(pos, np.float64).reshape(-1, 3)
        self.times = np.asarray(times, np.int64)
        self.n = len(self.pos)
        self.src, self.dst, self.ctimes = src, dst, ctimes
        self.m = len(src)
        self.R = np.tile(np.eye(3), (self.n, 1, 1))
        self.t = np.zeros((self.n, 3))
        self.nb = neighbours(self.n)
        self.enabled = self.times > last_deform_time
        self.e0 = int(np.argmax(self.enabled)) if self.enabled.any() else self.n
        self.N = self.n - self.e0
        self.cnode = np.zeros((self.m, K), np.int32)
        self.cw = np.zeros((self.m, K))
        for l in range(self.m):
            ids, w = weight_point(self.pos, self.times, self.src[l], int(self.ctimes[l]))
            self.cnode[l], self.cw[l] = ids, w
        self.cons_on = self.enabled[self.cnode].any(1)

    def vertex_position(self, l):
        p = np.zeros(3)
        s = self.src[l]
        for i in range(K):
            j, w = self.cnode[l, i], self.cw[l, i]
            d = s - self.pos[j]
            R = self.R[j]
            rd = np.array([R[q, 0] * d[0] + R[q, 1] * d[1] + R[q, 2] * d[2] for q in range(3)])
            p = p + w * ((rd + self.pos[j]) + self.t[j])
        return p

    def residual(self):
        r = []
        for j in range(self.n):
            if self.enabled[j]:
                c = self.R[j].T  # columns
                r += [c[0] @ c[1], c[0] @ c[2], c[1] @ c[2], c[0] @ c[0] - 1.0, c[1] @ c[1] - 1.0, c[2] @ c[2] - 1.0]
        sr = np.sqrt(W_REG)
        for j in range(self.n):
            for b in self.nb[j]:
                if self.enabled[j] or self.enabled[b]:
                    d = self.pos[b] - self.pos[j]
                    R = self.R[j]
                    rd = np.array([R[q, 0] * d[0] + R[q, 1] * d[1] + R[q, 2] * d[2] for q in range(3)])
                    r += list((((rd + self.pos[j]) + self.t[j]) - (self.pos[b] + self.t[b])) * sr)
        sc = np.sqrt(W_CON)
        for l in range(self.m):
            if self.cons_on[l]:
                r += list((self.vertex_position(l) - self.dst[l]) * sc)
        return np.array(r, np.float64)

    def jacobian(self):
        rows, cols, vals = [], [], []
        row = 0
        off = lambda j: (j - self.e0) * NV

        def put(r, c, v):
            rows.append(r); cols.append(c); vals.append(v)

        for j in range(self.n):
            if not self.enabled[j]:
                continue
            c0 = off(j)
            R = self.R[j]
            for i in range(3):
                put(row, c0 + i, R[i, 1]); put(row, c0 + 3 + i, R[i, 0])
                put(row + 1, c0 + i, R[i, 2]); put(row + 1, c0 + 6 + i, R[i, 0])
                put(row + 2, c0 + 3 + i, R[i, 2]); put(row + 2, c0 + 6 + i, R[i, 1])
                put(row + 3, c0 + i, 2 * R[i, 0]); put(row + 4, c0 + 3 + i, 2 * R[i, 1]); put(row + 5, c0 + 6 + i, 2 * R[i, 2])
            row += 6
        sr = np.sqrt(W_REG)
        for j in range(self.n):
            for b in self.nb[j]:
                if not (self.enabled[j] or self.enabled[b]):
                    continue
                d = self.pos[b] - self.pos[j]
                for q in range(3):
                    if self.enabled[b]:
                        put(row + q, off(b) + 9 + q, -1.0 * sr)
                    if self.enabled[j]:
                        for m in range(3):
                            put(row + q, off(j) + 3 * m + q, d[m] * sr)
                        put(row + q, off(j) + 9 + q, 1.0 * sr)
                row += 3
        sc = np.sqrt(W_CON)
        for l in range(self.m):
            if not self.cons_on[l]:
                continue
            for i in range(K):
                j, w = self.cnode[l, i], self.cw[l, i]
                if not self.enabled[j]:
                    continue
                d = (self.src[l] - self.pos[j]) * w
                for q in range(3):
                    for m in range(3):
                        put(row + q, off(j) + 3 * m + q, d[m] * sc)
                    put(row + q, off(j) + 9 + q, w * sc)
            row += 3
        return sp.csr_matrix((vals, (rows, cols)), shape=(row, NV * self.N))

    def solve_normal(self, J, r):
        """JᵀJ δ = -Jᵀr by band Cholesky in time order (LAPACK dpbtrf / dpbtrs)."""
        A = (J.T @ J).tocoo()
        g = -(J.T @ r)
        if A.shape[0] == 0:
            return g
        up = A.row <= A.col
        u = int((A.col[up] - A.row[up]).max())
        ab = np.zeros((u + 1, A.shape[0]))
        ab[u + A.row[up] - A.col[up], A.col[up]] = A.data[up]
        c = sla.cholesky_banded(ab, lower=False)
        return sla.cho_solve_banded((c, False), g)

    def apply(self, delta):
        for i in range(self.N):
            j = self.e0 + i
            dv = delta[NV * i:NV * i + NV]
            self.R[j] += dv[:9].reshape(3, 3).T  # column-major
            self.t[j] += dv[9:]

    def mean_cons_err(self):
        s = np.float32(0)
        for l in range(self.m):
            s = np.float32(np.float64(s) + _norm(self.vertex_position(l) - self.dst[l]))
        return np.float32(s / np.float32(self.m))

    def optimise(self):
        """optimiseGraphSparse (:416-492): returns dict(error, meanConsErr, iterations, stop)."""
        r = self.residual()
        J = self.jacobian()
        error = np.float32(r @ r)
        last = float(error)
        it, stop = 0, 0
        while it < 3:
            it += 1
            delta = self.solve_normal(J, r)
            self.apply(delta)
            r = self.residual()
            error = np.float32(r @ r)
            diff = float(error) - last
            dn = float(np.sqrt(delta @ delta))
            if float(error) > last:
                stop = 1
            elif dn < 1e-2:
                stop = 2
            elif float(error) < 1e-3:
                stop = 3
            elif abs(diff) < 1e-5 * float(error):
                stop = 4
            if stop:
                break
            last = float(error)
            J = self.jacobian()
        return dict(error=float(error), meanConsErr=float(self.mean_cons_err()), iterations=it, stop=stop)

    def nodes16(self):
        """Deformation.cpp:175-189: position, rotation column-major, translation, time; float32."""
        out = np.zeros((self.n, 16), np.float32)
        out[:, :3] = self.pos
        out[:, 3:12] = self.R.transpose(0, 2, 1).reshape(-1, 9)
        out[:, 12:15] = self.t
        out[:, 15] = self.times
        return out


def synthetic_case(n_nodes, n_cons, seed=0, shift=0.03):
    """A graph sampled along a closed camera loop (times ascending) and loop-closure-like constraints: the sources lie near
    the newest part of the map (time = the newest node's), the targets are the sources displaced by a small rigid motion
    and stamped with the time of an older part of the map. Returns (node_pos, node_times, src, dst, src_times, dst_times)."""
    rng = np.random.default_rng(seed)
    a = np.linspace(0, 2 * np.pi, n_nodes, endpoint=False)
    pos = np.stack([2 * np.cos(a), 2 * np.sin(a), 0.3 * np.sin(3 * a)], 1) + rng.normal(0, 0.15, (n_nodes, 3))
    times = np.sort(rng.integers(0, 20 * n_nodes, n_nodes)).astype(np.int32)
    newest = int(times[-1])
    near = rng.integers(max(0, n_nodes - 20), n_nodes, n_cons)
    src = pos[near] + rng.normal(0, 0.1, (n_cons, 3))
    th = 0.02
    Rz = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    dst = src @ Rz.T + np.array([shift, -shift / 2, shift / 3])
    dst_times = times[rng.integers(0, max(1, n_nodes // 2), n_cons)].astype(np.int32)
    return pos, times, src, dst, np.full(n_cons, newest, np.int32), dst_times


def deform_solve(node_pos, node_times, src, dst, src_times, dst_times=None, pin=False, last_deform_time=0):
    """Same arguments and results as elasticfusion_b200.capi.Context.deform_solve, plus the final R (n,3,3) and t (n,3) in
    float64: (info, nodes16, constraint nodes, constraint weights, R, t)."""
    S, D, T = expand_constraints(np.asarray(src).reshape(-1, 3), np.asarray(dst).reshape(-1, 3), src_times, dst_times, pin)
    s = Solver(node_pos, node_times, S, D, T, last_deform_time)
    info = s.optimise()
    info.update(n_nodes=s.n, n_enabled=s.N, n_constraints=s.m)
    return info, s.nodes16(), s.cnode, s.cw, s.R.copy(), s.t.copy()


REF_LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libef_refdef.so")


def ref_available():
    return os.path.exists(REF_LIB)


def ref_solve(node_pos, node_times, src, dst, src_times, dst_times=None, pin=False, last_deform_time=0):
    """The reference's own DeformationGraph + CholeskyDecomp (oracle/refdef, built into oracle/_ref/libef_refdef.so) on the
    same inputs as deform_solve: (info without stop / n_enabled, nodes16, constraint nodes, constraint weights, R, t)."""
    lib = C.CDLL(REF_LIB)
    pos = np.ascontiguousarray(node_pos, np.float64).reshape(-1, 3)
    nt = np.ascontiguousarray(node_times, np.int32)
    s = np.ascontiguousarray(src, np.float64).reshape(-1, 3)
    d = np.ascontiguousarray(dst, np.float64).reshape(-1, 3)
    st = np.ascontiguousarray(src_times, np.int32)
    dt = np.ascontiguousarray(st if dst_times is None else dst_times, np.int32)
    n, nc = len(pos), len(s)
    m = 2 * nc if pin else nc
    rt = np.zeros((n, 12)); nodes = np.zeros((n, 16), np.float32)
    cn = np.zeros((m, K), np.int32); cw = np.zeros((m, K))
    err, mce, it = C.c_float(), C.c_float(), C.c_int32()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.refdef_solve(p(pos), p(nt), n, p(s), p(d), p(st), p(dt), nc, int(pin), int(last_deform_time), p(rt), p(nodes), p(cn),
                          p(cw), C.byref(err), C.byref(mce), C.byref(it))
    assert rc == 0
    info = dict(error=float(err.value), meanConsErr=float(mce.value), iterations=it.value, n_nodes=n, n_constraints=m)
    R = rt[:, :9].reshape(n, 3, 3).transpose(0, 2, 1).copy()  # column-major -> R[i, row, col]
    return info, nodes, cn, cw, R, rt[:, 9:].copy()
