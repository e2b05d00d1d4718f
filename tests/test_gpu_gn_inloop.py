"""Every in-loop Gauss-Newton iteration of the tracker, entry by entry, against a float64 restatement of the reference at the
pose the device held.

The trace of ef_odom_track records, per iteration, the geometric and photometric systems the device reduced (A_icp, b_icp,
icp_residual, A_rgb, b_rgb, rgb_count, rgb_sigma, sigma_val) and the solve result; per SO(3) step, A_so3, b_so3 and
so3_residual. From the device's own earlier results this file rebuilds the pose every iteration started from, exactly as the
device forms it (gn_update_warp, so3_finish), evaluates the reference's per-pixel reductions at that pose from the pyramids the
device held (icpStep, computeRgbResidual + rgbStep, so3Step: Core/Cuda/reduce.cu, RGBDOdometry.cpp) and compares every entry.
Nothing drifts: iteration k is checked at the device's pose of iteration k, not at an oracle trajectory's.

The restatement runs every gate and projection in float32 as the kernels do and keeps every per-pixel term, so each entry's bar
is built from the terms:
- a pixel is *sure* when every gate decision and every nearest-pixel rounding it takes is more than delta from flipping, and
  *borderline* otherwise. delta is a running-error bound: each gated quantity q is re-evaluated with the absolute values of its
  operands (M_q), and delta_q = KAPPA * u * M_q, u = 2^-24. KAPPA = 32 covers two independent float32 evaluations of the longest
  chain (the geometric residual: two 3x3 transforms, two translations, a difference and a dot product, <= 13 roundings each,
  with or without FMA contraction) plus one ulp in every entry of the rebuilt float32 pose and warp matrices;
- |dev - sum_sure| <= sum_borderline max|term| + sum_sure err + c * eps32 * sum_all |term| per entry, where err is the same
  running-error bound carried through the row products, the borderline term is the largest over every rounding the pixel
  could take, and c = (rows a thread sums serially) + 16 covers the float32 summation tree (serial per thread, then shuffle
  and block trees of <= 9 levels, then the CTA partials in double, one product and one final rounding);
- counts (icp_residual[1], rgb_count, so3_residual[1]) and the integer rgb_sigma lie in [sum_sure, sum_sure + sum_borderline];
  sigma_val is the reference's expression of the device's own count and sigma, including its operator-precedence quirk.

The CPU test at the end pins the restatement to the oracle's stage functions, which test_oracle_golden.py / test_gpu_ref_pin.py
pin to the reference's own kernels."""
import math

import numpy as np
import pytest

from elasticfusion_b200 import capi, synth

gpu = pytest.mark.gpu
BIG = 2147483647 // 2
f32 = np.float32
U = 2.0 ** -24  # unit roundoff of float32
EPS32 = 2.0 ** -23
KAPPA = 32
DIST_THRES = f32(0.10)
ANGLE_THRES = f32(math.sin(f32(20.0) * f32(3.14159254) / f32(180.0)))
MAX_DEPTH_DELTA = f32(0.07)
SOBEL_SCALE = f32(0.125)
MIN_SCALE = (f32(1600.0), f32(576.0), f32(64.0))  # (minGrad / sobelScale)^2 for minGrad = 5, 3, 1 (RGBDOdometry.cpp:425)
PACK6 = [(i, j) for i in range(6) for j in range(i, 7)]  # JtJJtrSE3 order (types.cuh): upper triangle of [A | b]
PACK3 = [(i, j) for i in range(3) for j in range(i, 4)]  # JtJJtrSO3
GC_THREADS, IT1_THREADS, IT2_THREADS, RED_THREADS = 512, 128, 256, 256


# ---------------------------------------------------------------------------------------------------------------- restatement
def _terms(rows, err_rows, pack, extra):
    """Per-pixel products row_i * row_j in float64 (the packed system, then row_last^2, then `extra` columns) and their error
    bounds |r_i| e_j + |r_j| e_i."""
    r = rows.astype(np.float64)
    e = err_rows.astype(np.float64)
    last = r.shape[1] - 1
    cols = [r[:, i] * r[:, j] for i, j in pack] + [r[:, last] * r[:, last]]
    errs = [np.abs(r[:, i]) * e[:, j] + np.abs(r[:, j]) * e[:, i] for i, j in pack] + [2 * np.abs(r[:, last]) * e[:, last]]
    T = np.stack(cols + list(extra), 1)
    E = np.stack(errs + [np.zeros(len(r))] * len(extra), 1)
    return T, E


def _cross(a, b, s=-1.0):
    """a x b along axis 0; s = +1 gives the running-error magnitude of the same expression for non-negative operands."""
    return np.stack([a[1] * b[2] + s * a[2] * b[1], a[2] * b[0] + s * a[0] * b[2], a[0] * b[1] + s * a[1] * b[0]]).astype(a.dtype)


def _mv(M, v):
    """float32 3x3 times 3xN, each entry ((m0 v0 + m1 v1) + m2 v2) in the kernels' order"""
    return np.stack([(M[r, 0] * v[0] + M[r, 1] * v[1]) + M[r, 2] * v[2] for r in range(3)])


def _round_alt(q, r):
    """the other nearest integer q may round to"""
    return np.where(q >= r, r + 1, r - 1)


class Reduction:
    """The per-pixel terms of one reduction: `sure` (n_s, m) terms and `err` (n_s, m) bounds of the sure pixels, `border` (n_b, m)
    the largest |term| each borderline pixel can contribute. The last columns are counts (and, photometric, int(diff^2))."""

    def __init__(self, sure, err, border):
        self.sure, self.err, self.border = sure, err, border

    def sums(self):
        return self.sure.sum(0), self.err.sum(0), self.border.sum(0), np.abs(self.sure).sum(0) + self.border.sum(0)


def _classify(ev, n, ux, uy, qx, qy, dx, dy):
    """Runs evaluator ev(sel, ux, uy) -> (terms, err, strict, loose) at the nearest pixel and, for pixels whose rounding is
    within (dx, dy) of flipping, at every other pixel they may round to. Returns a Reduction."""
    sel = np.arange(n)
    T, E, strict, loose = ev(sel, ux, uy)
    rsure = (0.5 - np.abs(qx - ux) > dx) & (0.5 - np.abs(qy - uy) > dy)
    sure = rsure & strict
    bound = np.where(loose[:, None], np.abs(np.nan_to_num(T)), 0.0)
    maybe = loose.copy()
    rb = np.flatnonzero(~rsure)
    if len(rb):
        ax, ay = _round_alt(qx[rb], ux[rb]), _round_alt(qy[rb], uy[rb])
        xflip = 0.5 - np.abs(qx[rb] - ux[rb]) <= dx[rb]
        yflip = 0.5 - np.abs(qy[rb] - uy[rb]) <= dy[rb]
        for bx, by, ok in ((ax, uy[rb], xflip), (ux[rb], ay, yflip), (ax, ay, xflip & yflip)):
            T2, _, _, l2 = ev(rb, bx, by)
            l2 = l2 & ok
            bound[rb] = np.maximum(bound[rb], np.where(l2[:, None], np.abs(np.nan_to_num(T2)), 0.0))
            maybe[rb] |= l2
    border = ~sure & maybe & (~rsure | ~strict)
    return Reduction(T[sure], E[sure], bound[border])


def _in_range(ux, uy, cols, rows):
    return (ux >= 0) & (uy >= 0) & (ux < cols) & (uy < rows)


def _nearest(q):
    """__float2int_rn on finite values; non-finite ones land far outside any image"""
    return np.rint(np.where(np.isfinite(q), np.clip(q, -1e6, 1e6), -1e6)).astype(np.int64)


def icp_reduction(Rcurr, tcurr, Rprev_inv, tprev, vmap_curr, nmap_curr, vmap_g_prev, nmap_g_prev, fx, fy, cx, cy):
    """icpStep (reduce.cu ICPReduction::search / getProducts): live vertices to the world (Rcurr, tcurr), into the previous camera
    (Rprev_inv, tprev), projected with round-to-nearest; the world-frame model point and normal there; distance gate 0.1 and
    angle gate sin 20 deg; row [n, s x n, n.(s - d)] in the previous camera. Columns: 27 packed, row6^2, count."""
    rows, cols = vmap_curr.shape[0] // 3, vmap_curr.shape[1]
    Rcurr, tcurr, Rprev_inv, tprev = (np.asarray(a, f32) for a in (Rcurr, tcurr, Rprev_inv, tprev))
    fx, fy, cx, cy = (f32(v) for v in (fx, fy, cx, cy))
    v = vmap_curr.reshape(3, -1)
    nc = nmap_curr.reshape(3, -1)
    vg = vmap_g_prev.reshape(3, -1)
    ng = nmap_g_prev.reshape(3, -1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        live = np.flatnonzero(~np.isnan(v[0]))
        v, nc = v[:, live], nc[:, live]
        aR, aRi = np.abs(Rcurr), np.abs(Rprev_inv)
        s_g = _mv(Rcurr, v) + tcurr[:, None]
        M_sg = aR @ np.abs(v).astype(np.float64) + np.abs(tcurr)[:, None]
        s_cp = _mv(Rprev_inv, s_g - tprev[:, None])
        M_scp = aRi @ (M_sg + np.abs(tprev)[:, None])
        px = (s_cp[0] * fx) / s_cp[2] + cx
        py = (s_cp[1] * fy) / s_cp[2] + cy
        ux, uy = _nearest(px), _nearest(py)
        az = np.abs(s_cp[2]).astype(np.float64)
        dx = KAPPA * U * (fx * (M_scp[0] + np.abs(px - cx) / fx * M_scp[2]) / az + np.abs(px))
        dy = KAPPA * U * (fy * (M_scp[1] + np.abs(py - cy) / fy * M_scp[2]) / az + np.abs(py))
        keep = np.flatnonzero((s_cp[2] >= 0) & (ux >= -1) & (uy >= -1) & (ux <= cols) & (uy <= rows))
        s_g, M_sg, nc = s_g[:, keep], M_sg[:, keep], nc[:, keep]
        nc_g = _mv(Rcurr, nc)
        px, py, ux, uy, dx, dy = px[keep], py[keep], ux[keep], uy[keep], dx[keep], dy[keep]

    def ev(sel, bx, by):
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            inr = _in_range(bx, by, cols, rows)
            q = np.where(inr, by * cols + bx, 0)
            d = vg[:, q]
            n = ng[:, q]
            s, Ms, ncg = s_g[:, sel], M_sg[:, sel], nc_g[:, sel]
            e = d - s
            dist = np.sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2])
            cr = _cross(ncg, n)
            sine = np.sqrt(cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2])
            d_dist = KAPPA * U * (np.abs(d).sum(0) + Ms.sum(0) + dist)
            d_sine = KAPPA * U * 4.0
            finite = inr & ~np.isnan(nc[0, sel]) & ~np.isnan(n[0])
            strict = finite & (sine < ANGLE_THRES - d_sine) & (dist <= DIST_THRES - d_dist)
            loose = finite & (sine < ANGLE_THRES + d_sine) & (dist <= DIST_THRES + d_dist)
            s_cp = _mv(Rprev_inv, s - tprev[:, None])
            d_cp = _mv(Rprev_inv, d - tprev[:, None])
            n_cp = _mv(Rprev_inv, n)
            c = _cross(s_cp, n_cp)
            r6 = (n_cp[0] * (s_cp[0] - d_cp[0]) + n_cp[1] * (s_cp[1] - d_cp[1])) + n_cp[2] * (s_cp[2] - d_cp[2])
            M_s = aRi @ (Ms + np.abs(tprev)[:, None])
            M_d = aRi @ (np.abs(d).astype(np.float64) + np.abs(tprev)[:, None])
            M_n = aRi @ np.abs(n).astype(np.float64)
            M_c = _cross(M_s, M_n, 1.0)
            M_6 = (M_n * (M_s + M_d)).sum(0)
            row = np.stack([n_cp[0], n_cp[1], n_cp[2], c[0], c[1], c[2], r6], 1)
            M = np.stack([M_n[0], M_n[1], M_n[2], M_c[0], M_c[1], M_c[2], M_6], 1)
            T, E = _terms(row, KAPPA * U * M, PACK6, [np.ones(len(sel))])
        return T, E, strict, loose

    return _classify(ev, len(keep), ux, uy, px, py, dx, dy)


GSX = np.array([0.52201, 0.00000, -0.52201, 0.79451, -0.00000, -0.79451, 0.52201, 0.00000, -0.52201], f32)
GSY = np.array([0.52201, 0.79451, 0.52201, 0.00000, 0.00000, 0.00000, -0.52201, -0.79451, -0.52201], f32)


def sobel(img):
    """computeDerivativeImages (cudafuncs.cu applyKernel): float32 sums in the kernel's order, truncated to int16. At the border
    the kernel index keeps counting down over the clipped window, as the reference's loop does."""
    rows, cols = img.shape
    src = img.astype(f32)
    dx = np.zeros((rows, cols), f32)
    dy = np.zeros((rows, cols), f32)
    k = 8
    pad = np.pad(src, 1)
    for j in (-1, 0, 1):
        for i in (-1, 0, 1):
            s = pad[1 + j:1 + j + rows, 1 + i:1 + i + cols]
            dx = dx + s * GSX[k]
            dy = dy + s * GSY[k]
            k -= 1
    for y, x in zip(*np.nonzero(_border_mask(rows, cols))):
        ax, ay, kk = f32(0), f32(0), 8
        for jj in range(max(y - 1, 0), min(y + 1, rows - 1) + 1):
            for ii in range(max(x - 1, 0), min(x + 1, cols - 1) + 1):
                ax = f32(ax + f32(src[jj, ii] * GSX[kk]))
                ay = f32(ay + f32(src[jj, ii] * GSY[kk]))
                kk -= 1
        dx[y, x], dy[y, x] = ax, ay
    return np.trunc(dx).astype(np.int32).astype(np.int16), np.trunc(dy).astype(np.int32).astype(np.int16)


def _border_mask(rows, cols):
    m = np.zeros((rows, cols), bool)
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = True
    return m


def rgb_candidates(level, dIdx, dIdy, next_depth, next_image):
    """The pose-independent gates of computeRgbResidual: j < cols-5, i < rows-1, the 4x4 window [i-2, i+2) x [j-2, j+2) of the
    live image non-zero, |gradient|^2 >= minScale, live depth finite. Returns (y, x) of the candidates."""
    rows, cols = next_image.shape
    ok = np.zeros((rows, cols), bool)
    ok[:rows - 1, :cols - 5] = True
    pos = next_image > 0
    win = np.ones((rows, cols), bool)
    for du in (-2, -1, 0, 1):
        for dv in (-2, -1, 0, 1):
            sh = np.ones((rows, cols), bool)
            ys = slice(max(-du, 0), rows - max(du, 0))
            xs = slice(max(-dv, 0), cols - max(dv, 0))
            sh[ys, xs] = pos[max(du, 0):rows + min(du, 0), max(dv, 0):cols + min(dv, 0)]
            win &= sh
    m2 = (dIdx.astype(np.int32) ** 2 + dIdy.astype(np.int32) ** 2).astype(f32)
    ok &= win & (m2 >= MIN_SCALE[level]) & ~np.isnan(next_depth)
    return np.nonzero(ok)


def rgb_reduction(level, krkinv, kt, sigma, dIdx, dIdy, last_depth, next_depth, last_image, next_image, fx, fy, cx, cy):
    """computeRgbResidual (reduce.cu RGBResidual::getProducts) at the warp (krkinv, kt) and rgbStep (RGBReduction::getProducts)
    with weight sigma on the correspondences it finds; the cloud point is projectPoints' of lastDepth at the model pixel.
    Columns: 27 packed, row6^2, count, int(diff^2)."""
    rows, cols = next_image.shape
    k, t = np.asarray(krkinv, f32).reshape(3, 3), np.asarray(kt, f32)
    fx, fy, cx, cy = (f32(v) for v in (fx, fy, cx, cy))
    sigma = f32(sigma)
    ys, xs = rgb_candidates(level, dIdx, dIdy, next_depth, next_image)
    x, y = xs.astype(f32), ys.astype(f32)
    d1 = next_depth[ys, xs]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        num = [d1 * ((k[r, 0] * x + k[r, 1] * y) + k[r, 2]) + t[r] for r in range(3)]
        Mn = [d1.astype(np.float64) * (abs(k[r, 0]) * x + abs(k[r, 1]) * y + abs(k[r, 2])) + abs(t[r]) for r in range(3)]
        td = num[2]
        qx, qy = num[0] / td, num[1] / td
        ux, uy = _nearest(qx), _nearest(qy)
        atd = np.abs(td).astype(np.float64)
        dx = KAPPA * U * ((Mn[0] + np.abs(qx) * Mn[2]) / atd + np.abs(qx))
        dy = KAPPA * U * ((Mn[1] + np.abs(qy) * Mn[2]) / atd + np.abs(qy))
    inv_fx, inv_fy = f32(1.0) / fx, f32(1.0) / fy
    gxs, gys = dIdx[ys, xs].astype(f32), dIdy[ys, xs].astype(f32)
    live = next_image[ys, xs].astype(f32)

    def ev(sel, bx, by):
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            inr = _in_range(bx, by, cols, rows)
            q0, q1 = np.where(inr, by, 0), np.where(inr, bx, 0)
            d0 = last_depth[q0, q1]
            li = last_image[q0, q1]
            gap = np.abs(td[sel] - d0)
            dg = KAPPA * U * (Mn[2][sel] + np.abs(d0))
            base = inr & (d0 > 0) & (li != 0)
            strict = base & (gap <= MAX_DEPTH_DELTA - dg)
            loose = base & (gap <= MAX_DEPTH_DELTA + dg)
            diff = live[sel] - li.astype(f32)
            sq = np.trunc(diff * diff).astype(np.float64)
            w = sigma + np.abs(diff)
            w = np.where(w > f32(1.19209290e-07), f32(1.0) / w, f32(1.0)).astype(f32)
            if sigma == -1:
                w = np.ones_like(w)
            r6 = -w * diff
            cpx = ((bx.astype(f32) - cx) * d0) * inv_fx
            cpy = ((by.astype(f32) - cy) * d0) * inv_fy
            cpz = d0
            invz = (1.0 / cpz.astype(np.float64)).astype(f32)
            v0 = ((w * SOBEL_SCALE) * gxs[sel] * fx) * invz
            v1 = ((w * SOBEL_SCALE) * gys[sel] * fy) * invz
            v2 = -(v0 * cpx + v1 * cpy) * invz
            row = np.stack([v0, v1, v2, -cpz * v1 + cpy * v2, cpz * v0 - cpx * v2, -cpy * v0 + cpx * v1, r6], 1)
            a0, a1, ax_, ay_, az_ = (np.abs(a).astype(np.float64) for a in (v0, v1, cpx, cpy, cpz))
            a2 = (a0 * ax_ + a1 * ay_) * np.abs(invz)
            M = np.stack([a0, a1, a2, az_ * a1 + ay_ * a2, az_ * a0 + ax_ * a2, ay_ * a0 + ax_ * a1, np.abs(r6)], 1)
            T, E = _terms(row, KAPPA * U * M, PACK6, [np.ones(len(sel)), sq])
        return T, E, strict, loose

    return _classify(ev, len(xs), ux, uy, qx, qy, dx, dy)


def so3_reduction(last_image, next_image, image_basis, kinv, krlr):
    """so3Step (reduce.cu SO3Reduction::getProducts): the pixel warped by the homography, rounded to nearest, both pixels one
    away from the border; gradients of both images averaged; row [(leftProduct x point), -(next - last)].
    Columns: 9 packed, row3^2, count."""
    rows, cols = next_image.shape
    H, Ki, Kr = (np.asarray(m, f32).reshape(3, 3) for m in (image_basis, kinv, krlr))
    ys, xs = np.nonzero(np.ones((rows, cols), bool))
    x, y, one = xs.astype(f32), ys.astype(f32), np.ones(len(xs), f32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        w = _mv(H, np.stack([x, y, one]))
        Mw = np.abs(H).astype(np.float64) @ np.stack([x, y, one]).astype(np.float64)
        qx, qy = w[0] / w[2], w[1] / w[2]
        ux, uy = _nearest(qx), _nearest(qy)
        aw = np.abs(w[2]).astype(np.float64)
        dx = KAPPA * U * ((Mw[0] + np.abs(qx) * Mw[2]) / aw + np.abs(qx))
        dy = KAPPA * U * ((Mw[1] + np.abs(qy) * Mw[2]) / aw + np.abs(qy))
    nxt, lst = next_image.astype(f32), last_image.astype(f32)
    inner = (xs >= 1) & (xs < cols - 1) & (ys >= 1) & (ys < rows - 1)
    p = _mv(Ki, np.stack([x, y, one]))
    Mp = np.abs(Ki).astype(np.float64) @ np.stack([x, y, one]).astype(np.float64)
    two = f32(2.0)

    def grad(img, gx_, gy_):
        actu = img[gy_, gx_]
        gx = ((img[gy_, gx_ - 1] + actu) / two) - ((img[gy_, gx_ + 1] + actu) / two)
        gy = ((img[gy_ - 1, gx_] + actu) / two) - ((img[gy_ + 1, gx_] + actu) / two)
        return gx, gy

    def ev(sel, bx, by):
        ok = inner[sel] & (bx >= 1) & (bx < cols - 1) & (by >= 1) & (by < rows - 1)
        cbx, cby = np.where(ok, bx, 1), np.where(ok, by, 1)
        cx_, cy_ = np.where(ok, xs[sel], 1), np.where(ok, ys[sel], 1)
        gnx, gny = grad(nxt, cbx, cby)
        glx, gly = grad(lst, cx_, cy_)
        gx, gy = (gnx + glx) / two, (gny + gly) / two
        pp, Mpp = p[:, sel], Mp[:, sel]
        xx, yy = x[sel], y[sel]
        z2 = pp[2] * pp[2]
        a, b, c, d, e, f, g, h, i = (Kr[r, cc] for r in range(3) for cc in range(3))
        lp = np.stack([((pp[2] * (d * gy + a * gx)) - (gy * g * yy) - (gx * g * xx)) / z2,
                       ((pp[2] * (e * gy + b * gx)) - (gy * h * yy) - (gx * h * xx)) / z2,
                       ((pp[2] * (f * gy + c * gx)) - (gy * i * yy) - (gx * i * xx)) / z2])
        A = np.abs
        agx, agy = A(gx).astype(np.float64), A(gy).astype(np.float64)
        Mz2 = Mpp[2] * Mpp[2]
        Mlp = np.stack([(Mpp[2] * (A(d) * agy + A(a) * agx) + agy * A(g) * yy + agx * A(g) * xx + A(lp[0]) * Mz2) / z2,
                        (Mpp[2] * (A(e) * agy + A(b) * agx) + agy * A(h) * yy + agx * A(h) * xx + A(lp[1]) * Mz2) / z2,
                        (Mpp[2] * (A(f) * agy + A(c) * agx) + agy * A(i) * yy + agx * A(i) * xx + A(lp[2]) * Mz2) / z2])
        jac = _cross(lp, pp)
        Mjac = _cross(Mlp, Mpp, 1.0)
        r3 = -(nxt[cby, cbx] - lst[cy_, cx_])
        row = np.where(ok[:, None], np.stack([jac[0], jac[1], jac[2], r3], 1), f32(0))
        M = np.stack([Mjac[0], Mjac[1], Mjac[2], np.zeros(len(sel))], 1)
        T, E = _terms(row, KAPPA * U * M, PACK3, [ok.astype(np.float64)])
        return T, E, ok, ok

    return _classify(ev, len(xs), ux, uy, qx, qy, dx, dy)


# ---------------------------------------------------------------------------------------------------------- checking the bars
def check_entries(what, dev, red: Reduction, c, counts=()):
    """dev: the device's packed values in the Reduction's column order (None where not compared). `counts`: indices of the
    integer-valued columns (bounded by [sure, sure + borderline]). Returns (largest |dev - ref| / bound, borderline count)."""
    S, E, B, Aall = red.sums()
    worst = 0.0
    for k, v in enumerate(dev):
        if v is None:
            continue
        if k in counts:
            assert S[k] <= v <= S[k] + B[k], (what, "count", k, v, S[k], B[k])
            continue
        bound = B[k] + E[k] + c * EPS32 * Aall[k]
        gap = abs(float(v) - S[k])
        assert gap <= bound, (what, k, float(v), S[k], gap, bound)
        if bound > 0:
            worst = max(worst, gap / bound)
    return worst, len(red.border)


def packed_from_system(A, b, pack):
    n = len(b)
    return [b[i] if j == n else A[i, j] for i, j in pack]


# ------------------------------------------------------------------------------------------------------------- pose rebuild
def rodrigues(r):
    R = np.eye(3)
    theta = float(np.sqrt(r @ r))
    if theta >= np.finfo(np.float64).eps:
        c, s = np.cos(theta), np.sin(theta)
        k = r / theta
        kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        R = c * np.eye(3) + (1.0 - c) * np.outer(k, k) + s * kx
    return R


def level_K(K, lv):
    """K and its closed-form inverse of pyramid level lv in double, from the float level intrinsics (CameraModel(level))"""
    fx, fy, cx, cy = (float(f32(v) / f32(1 << lv)) for v in (K.fx, K.fy, K.cx, K.cy))
    Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    Ki = np.array([[1 / fx, 0, -cx / fx], [0, 1 / fy, -cy / fy], [0, 0, 1.0]])
    return Km, Ki, (fx, fy, cx, cy)


def warp_of(resultRt, K, lv):
    """KRK^-1 and K t of resultRt^-1 = [R^T | -R^T t] in double, then cast (RGBDOdometry.cpp:407-417)"""
    Km, Ki, _ = level_K(K, lv)
    R = resultRt[:3, :3].T
    t = -(R @ resultRt[:3, 3])
    return (Km @ R @ Ki).astype(f32), (Km @ t).astype(f32)


def curr_of(resultRt, Rprev, tprev):
    """currentT = T_prev * rgbOdom^-1 in float (RGBDOdometry.cpp:543-551): iR = R^T, it = -(iR t)"""
    iR = resultRt[:3, :3].T.astype(f32)
    ot = resultRt[:3, 3].astype(f32)
    it = -_mv(iR, ot[:, None])[:, 0]
    return _mv(Rprev, iR).astype(f32), (_mv(Rprev, it[:, None])[:, 0] + tprev).astype(f32)


def so3_poses(so3_records):
    """resultR for every SO(3) record and the one the SE(3) loop starts from, chained as so3_finish does: convergence / divergence
    tests on sqrt(res0)/res1 in float, delta from the 3x3 system, R_lr = float(rodrigues(delta)) * R_lr in float."""
    R_lr = np.eye(3, dtype=f32)
    last_err, last_cnt = f32(np.finfo(f32).max / 2), f32(np.finfo(f32).max / 2)
    last_R = R_lr.copy()
    used = []
    for t in so3_records:
        used.append(R_lr.astype(np.float64))
        res = t["so3_residual"]
        err = f32(np.sqrt(f32(res[0])) / f32(res[1]))
        if err < last_err and last_cnt == f32(res[1]):
            return used, R_lr.astype(np.float64)
        if float(err) > float(last_err) + 0.001:
            return used, last_R.astype(np.float64)
        last_err, last_cnt, last_R = err, f32(res[1]), R_lr.copy()
        A = t["A_so3"].astype(np.float64).reshape(3, 3)
        delta = np.linalg.solve(A, t["b_so3"].astype(np.float64)).astype(f32)
        R_lr = (rodrigues(delta.astype(np.float64)).astype(f32) @ R_lr).astype(f32)
    return used, R_lr.astype(np.float64)


# ----------------------------------------------------------------------------------------------------------- device harness
SIZES = {
    "640x480": synth.K_DEFAULT,
    "424x240": synth.Intrinsics(424, 240, 212.0, 212.0, 212.0, 120.0),  # level-2 width 106: a partial 4-pixel group
    "480x270": synth.Intrinsics(480, 270, 240.0, 240.0, 240.0, 135.0),  # odd row counts at levels 1 (135) and 2 (67)
    "1920x1080": synth.Intrinsics(1920, 1080, 960.0, 960.0, 960.0, 540.0),
}
# EF_GN_CLUSTER (cluster size, 0 = two-kernel path) and EF_GN_CLUSTER_LEVELS (coarse levels inside the cluster launch)
PATHS = {"cluster": (None, None), "cluster-3lv": (None, "3"), "cluster8": ("8", None), "two-kernel": ("0", None)}
TRACKERS = {
    "default": dict(so3=False),
    "so3": dict(so3=True),
    "rgb_only": dict(rgb_only=True, so3=False),
    "icp_w100": dict(icp_weight=100.0, so3=False),
    "fast_odom": dict(fast_odom=True, so3=False),
    "no_pyramid": dict(pyramid=False, so3=False),
}
CASES = [(s, p, t) for s in ("640x480", "424x240") for p in PATHS for t in TRACKERS] + \
        [(s, p, "default") for s in ("480x270", "1920x1080") for p in ("cluster", "two-kernel")]
_FRAMES = {}


def _frames(size):
    if size not in _FRAMES:
        _FRAMES[size] = list(synth.sequence(4, SIZES[size], seed=42, noise=True))
    return _FRAMES[size]


def _device_run(size, path, cfg, monkeypatch):
    """Three frames through ef_process_frame, then the init stages for frame 3 from the model's FILL_* buffers and one
    ef_odom_track. Returns (T_prev, trace, pyramids as the device held them before the call, DIDX/DIDY after it)."""
    from oracle import ef_oracle as eo
    from util import rgba_of

    K = SIZES[size]
    cl, lv = PATHS[path]
    for var, val in (("EF_GN_CLUSTER", cl), ("EF_GN_CLUSTER_LEVELS", lv)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)
    frames = _frames(size)
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=3 * K.width * K.height, time_delta=BIG))
    try:
        for i in range(3):
            ctx.process_frame(frames[i][0], frames[i][1], i)
        T_prev = ctx.get_pose()
        rgb, depth, _ = frames[3]
        ctx.upload("DEPTH_FILTERED", eo.bilateral(depth, 3.0))
        ctx.upload("RGBA", rgba_of(rgb))
        ctx.odom_init_icp_model(ctx.buffer_ptr("FILL_VERTEX")[0], ctx.buffer_ptr("FILL_NORMAL")[0], T_prev)
        ctx.odom_init_rgb_model(ctx.buffer_ptr("FILL_IMAGE")[0])
        ctx.odom_init_icp_depth(ctx.buffer_ptr("DEPTH_FILTERED")[0], 20.0)
        ctx.odom_init_rgb(ctx.buffer_ptr("RGBA")[0])
        names = ("VMAP_CURR", "NMAP_CURR", "VMAP_G_PREV", "NMAP_G_PREV", "LAST_DEPTH", "NEXT_DEPTH", "LAST_IMAGE", "NEXT_IMAGE",
                 "LAST_NEXT_IMAGE")
        pyr = {(n, l): ctx.download(n, l) for n in names for l in range(3)}  # before odom_track: SO(3) swaps the image handles
        T_out, trace = ctx.odom_track(T_prev, **cfg)
        sob = {l: (ctx.download("DIDX", l), ctx.download("DIDY", l)) for l in range(3)}
    finally:
        ctx.close()
    return T_prev, trace, pyr, sob


def _red_blocks(n_items, per_thread, threads, ctas_per_sm, sms):
    b = -(-n_items // (threads * per_thread))
    cap = min(sms * ctas_per_sm, 1184)
    if b > cap:
        rounds = -(-b // cap)
        b = -(-b // rounds)
    return max(b, 1)


def _serial(size, path, lv, n_icp, n_rgb, sms):
    """rows one thread sums serially in the pass that reduced level lv: (geometric, photometric)"""
    K = SIZES[size]
    rows, cols = K.height >> lv, K.width >> lv
    N = rows * cols
    cl, levels = PATHS[path]
    in_cluster = cl != "0" and lv >= 3 - int(levels or 1)
    per = 4 if cols % 4 == 0 else 1
    if in_cluster:
        T = int(cl or 8) * GC_THREADS  # 16 CTAs when the device can co-schedule them; 8 bounds both
        return per * -(-N // (per * T)), -(-n_rgb // T)
    nb1 = _red_blocks(N, 4, IT1_THREADS, 5, sms)
    nb2 = min(max(max(N // 8 + IT2_THREADS - 1, 0) // IT2_THREADS, (nb1 + 7) // 8, 1), 160)
    return per * -(-N // (per * nb1 * IT1_THREADS)), -(-n_rgb // (nb2 * IT2_THREADS))


@gpu
@pytest.mark.parametrize("size,path,tracker", CASES, ids=["-".join(c) for c in CASES])
def test_inloop_systems_match_float64_reference(size, path, tracker, monkeypatch):
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    K = SIZES[size]
    cfg = TRACKERS[tracker]
    T_prev, trace, pyr, sob = _device_run(size, path, cfg, monkeypatch)
    w = float(cfg.get("icp_weight", 10.0))
    rgb_only = cfg.get("rgb_only", False)
    icp_on, rgb_on = (not rgb_only) and w > 0, rgb_only or w < 100
    Rprev, tprev = T_prev[:3, :3].astype(f32), T_prev[:3, 3].astype(f32)
    Rprev_inv = np.linalg.inv(Rprev.astype(np.float64)).astype(f32)
    worst, border = 0.0, 0

    # Sobel images of the live pyramid: bit-exact (the photometric gates and rows read them)
    dI = {}
    if rgb_on:
        for lv in range(3):
            dI[lv] = sobel(pyr[("NEXT_IMAGE", lv)])
            assert (dI[lv][0] == sob[lv][0]).all() and (dI[lv][1] == sob[lv][1]).all(), ("sobel", lv)

    so3 = [t for t in trace if t["kind"] == 1]
    se3 = [t for t in trace if t["kind"] == 0]
    assert bool(so3) == bool(cfg.get("so3", True))
    resultR = np.eye(3)
    if so3:
        Km, Ki, _ = level_K(K, 2)
        used, resultR = so3_poses(so3)
        n2 = (K.height >> 2) * (K.width >> 2)
        for t, R in zip(so3, used):
            red = so3_reduction(pyr[("LAST_NEXT_IMAGE", 2)], pyr[("NEXT_IMAGE", 2)], (Km @ R @ Ki).astype(f32), Ki.astype(f32),
                                (Km @ R).astype(f32))
            T_so3 = int(PATHS[path][0] or 8) * GC_THREADS if PATHS[path][0] != "0" else _red_blocks(n2, 1, RED_THREADS, 2, sms) * RED_THREADS
            A, b = t["A_so3"].reshape(3, 3), t["b_so3"]
            dev = packed_from_system(A, b, PACK3) + [t["so3_residual"][0], t["so3_residual"][1]]
            r, nb = check_entries((size, path, tracker, "so3", int(t["iter"])), dev, red, -(-n2 // T_so3) + 16 + 16, counts=(10,))
            worst, border = max(worst, r), max(border, nb)

    # SE(3): the pose each iteration started from, from the device's own earlier results
    expected = [(lv, it) for lv, n in ((2, 4 if cfg.get("pyramid", True) else 0), (1, 5 if cfg.get("pyramid", True) else 0),
                                       (0, 3 if cfg.get("fast_odom") else 10)) for it in range(n)]
    got = [(int(t["level"]), int(t["iter"])) for t in se3]
    if rgb_only:  # the photometric-only `break` ends a level early
        assert all(g in expected for g in got) and got == sorted(got, key=expected.index), got
    else:
        assert got == expected, got
    resultRt = np.eye(4)
    resultRt[:3, :3] = resultR
    Rcurr, tcurr = Rprev.copy(), tprev.copy()
    for t in se3:
        lv, it = int(t["level"]), int(t["iter"])
        where = (size, path, tracker, lv, it)
        _, _, (fx, fy, cx, cy) = level_K(K, lv)
        fx, fy, cx, cy = (f32(v) for v in (fx, fy, cx, cy))
        A_icp, b_icp = t["A_icp"].reshape(6, 6), t["b_icp"]
        A_rgb, b_rgb = t["A_rgb"].reshape(6, 6), t["b_rgb"]
        if icp_on:
            red = icp_reduction(Rcurr, tcurr, Rprev_inv, tprev, pyr[("VMAP_CURR", lv)], pyr[("NMAP_CURR", lv)], pyr[("VMAP_G_PREV", lv)],
                                pyr[("NMAP_G_PREV", lv)], fx, fy, cx, cy)
            n_icp = (K.height >> lv) * (K.width >> lv)
            ser = _serial(size, path, lv, n_icp, n_icp, sms)[0]
            dev = packed_from_system(A_icp, b_icp, PACK6) + [t["icp_residual"][0], t["icp_residual"][1]]
            r, nb = check_entries(where + ("icp",), dev, red, ser + 16, counts=(28,))
            worst, border = max(worst, r), max(border, nb)
        else:
            assert not A_icp.any() and not b_icp.any(), where
        if rgb_on:
            krkinv, kt = warp_of(resultRt, K, lv)
            cnt, sig, sv = int(t["rgb_count"]), int(t["rgb_sigma"]), float(t["sigma_val"])
            # sigmaVal = sqrt((float)sigma / rgbSize == 0 ? 1 : rgbSize) (RGBDOdometry.cpp:442), -1 when photometric-only
            quirk = f32(math.sqrt(1 if (cnt and sig == 0) else cnt)) if cnt else f32(0.0)
            assert sv == (-1.0 if rgb_only else float(quirk)), (where, "sigma_val", sv, cnt, sig)
            red = rgb_reduction(lv, krkinv, kt, sv, dI[lv][0], dI[lv][1], pyr[("LAST_DEPTH", lv)], pyr[("NEXT_DEPTH", lv)],
                                pyr[("LAST_IMAGE", lv)], pyr[("NEXT_IMAGE", lv)], fx, fy, cx, cy)
            ser = _serial(size, path, lv, 0, len(red.sure) + len(red.border), sms)[1]
            dev = packed_from_system(A_rgb, b_rgb, PACK6) + [None, cnt, sig]
            r, nb = check_entries(where + ("rgb",), dev, red, ser + 16, counts=(28, 29))
            worst, border = max(worst, r), max(border, nb)
        else:
            assert not A_rgb.any() and not b_rgb.any() and int(t["rgb_count"]) == 0, where
        # the recorded system and its solve (the in-loop gather of the packed sums feeds the solve, not the record)
        lastA, lastb, x = t["lastA"].reshape(6, 6), t["lastb"], t["result"]
        Ai, Ar = A_icp.astype(np.float64), A_rgb.astype(np.float64)
        bi, br = b_icp.astype(np.float64), b_rgb.astype(np.float64)
        A_ref = Ar + w * w * Ai if (icp_on and rgb_on) else (Ai if icp_on else Ar)
        b_ref = br + w * bi if (icp_on and rgb_on) else (bi if icp_on else br)
        assert (np.abs(lastA - A_ref) <= 1e-12 * np.abs(A_ref)).all() and (np.abs(lastb - b_ref) <= 1e-12 * np.abs(b_ref)).all(), where
        x_ref = np.linalg.solve(lastA, lastb)
        assert np.abs(x - x_ref).max() <= np.linalg.cond(lastA) * 1e-14 * np.abs(x_ref).max(), (where, "solve", x, x_ref)
        inc = np.eye(4)
        inc[:3, :3] = rodrigues(np.asarray(x[3:], np.float64))
        inc[:3, 3] = x[:3]
        resultRt = inc @ resultRt
        Rcurr, tcurr = curr_of(resultRt, Rprev, tprev)
    print(f"\ninloop {size} {path} {tracker}: max |dev-ref|/bound {worst:.3f}, max borderline pixels {border}")


# ----------------------------------------------------------------------------------------------------------------- CPU pin
def test_restatement_matches_oracle_stage_functions(frames, K):
    """The restatement against the oracle's icp_step, rgb_residual + rgb_step and so3_step on identical inputs and the same
    bars (the oracle sums float32 products in double: c = 4)."""
    from oracle import ef_oracle as eo
    from util import rgba_of, run_oracle

    f = run_oracle(frames, K, 3)
    rgb, depth, _ = frames[3]
    od = f.odometry()
    T = f.pose
    od.init_icp_model(f.buffer("fill_vertex"), f.buffer("fill_normal"), T)
    od.init_rgb_model(f.buffer("fill_image"))
    od.init_icp_depth(eo.bilateral(depth, 3.0), 20.0)
    od.init_rgb(rgba_of(rgb))
    R, t = T[:3, :3].astype(f32), T[:3, 3].astype(f32)
    dR = rodrigues(np.array([0.003, -0.002, 0.0015]))
    Rcurr, tcurr = (R @ dR.astype(f32)).astype(f32), (t + np.array([0.004, -0.003, 0.005], f32)).astype(f32)
    Rprev_inv = np.linalg.inv(R.astype(np.float64)).astype(f32)
    for lv in range(3):
        Km, Ki, (fx, fy, cx, cy) = level_K(K, lv)
        fx, fy, cx, cy = (f32(v) for v in (fx, fy, cx, cy))
        vc, nc, vg, ng = (od.buffer(n, lv) for n in ("vmap_curr", "nmap_curr", "vmap_g_prev", "nmap_g_prev"))
        Ao, bo, ro = eo.icp_step(Rcurr, tcurr, vc, nc, Rprev_inv, t, fx, fy, cx, cy, vg, ng, float(DIST_THRES), float(ANGLE_THRES))
        red = icp_reduction(Rcurr, tcurr, Rprev_inv, t, vc, nc, vg, ng, fx, fy, cx, cy)
        _, nb = check_entries(("icp", lv), packed_from_system(Ao, bo, PACK6) + [ro[0], ro[1]], red, 4, counts=(28,))
        assert len(red.sure) > 1000 and nb <= max(10, len(red.sure) // 100), (lv, len(red.sure), nb)

        nI = od.buffer("nextImage", lv)
        dIdx, dIdy = eo.sobel(nI)
        sx, sy = sobel(nI)
        assert (sx == dIdx).all() and (sy == dIdy).all(), ("sobel", lv)
        inc = np.eye(4)
        inc[:3, :3] = rodrigues(np.array([0.002, 0.003, -0.001]))
        inc[:3, 3] = [0.004, -0.002, 0.003]
        krkinv, kt = warp_of(inc, K, lv)
        ld, nd, li = od.buffer("lastDepth", lv), od.buffer("nextDepth", lv), od.buffer("lastImage", lv)
        corres, sig, cnt = eo.rgb_residual(MIN_SCALE[lv], dIdx, dIdy, ld, nd, li, nI, float(MAX_DEPTH_DELTA), kt, krkinv)
        sigma = float(f32(math.sqrt(cnt)))
        Ao, bo = eo.rgb_step(corres, sigma, eo.project_points(ld, fx, fy, cx, cy), fx, fy, dIdx, dIdy, float(SOBEL_SCALE))
        red = rgb_reduction(lv, krkinv, kt, sigma, dIdx, dIdy, ld, nd, li, nI, fx, fy, cx, cy)
        _, nb = check_entries(("rgb", lv), packed_from_system(Ao, bo, PACK6) + [None, cnt, sig], red, 4, counts=(28, 29))
        assert len(red.sure) > 100 and nb <= max(10, len(red.sure) // 100), (lv, len(red.sure), nb)

    Km, Ki, _ = level_K(K, 2)
    Rs = rodrigues(np.array([0.004, -0.003, 0.002]))
    H, kinv, krlr = (Km @ Rs @ Ki).astype(f32), Ki.astype(f32), (Km @ Rs).astype(f32)
    Ao, bo, ro = eo.so3_step(od.buffer("lastNextImage", 2), od.buffer("nextImage", 2), H, kinv, krlr)
    red = so3_reduction(od.buffer("lastNextImage", 2), od.buffer("nextImage", 2), H, kinv, krlr)
    _, nb = check_entries("so3", packed_from_system(Ao, bo, PACK3) + [ro[0], ro[1]], red, 4, counts=(10,))
    assert len(red.sure) > 1000 and nb <= max(10, len(red.sure) // 100), (len(red.sure), nb)
