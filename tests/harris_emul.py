"""numpy emulation of the fused Harris kernel's arithmetic (image_b200/csrc/harris_kernels3.cuh) and of its
error bound harris_eps, operation by operation, for frames interior to the image (no border logic): used on the CPU
to check that the bound really bounds |R_fp32 - R_reference| (tests/test_harris_certify_cpu.py).

fma(a, b, c) is emulated as float32(float64(a) * float64(b) + float64(c)): the product of two floats is exact in
double, the sum is rounded to double and then to float (double rounding differs from a true FMA in ~1e-9 of the
cases by half an ulp - irrelevant for a bound with a 25 % margin).
"""
import numpy as np

F = np.float32
U = F(5.9604645e-8)


def taps(sigma):
    """gaussian.cpp:306-329 in double; the half-width (int)(3 * sigma) is a float32 product there."""
    size = int(F(3) * F(sigma)) + 1
    den = float(F(2) * F(sigma) * F(sigma))
    s = float(F(sigma))
    B = np.array([1 / (s * np.sqrt(2.0 * 3.1415926)) * np.exp(-i * i / den) for i in range(size)])
    norm = B.sum() * 2 - B[0]
    return B / norm


def fma(a, b, c):
    return (a.astype(np.float64) * np.float64(b) + c.astype(np.float64)).astype(F) if np.isscalar(b) or np.ndim(b) == 0 \
        else (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F)


def shift(a, dy, dx):
    """a[y+dy, x+dx] with wrap-around (callers crop the border away)."""
    return np.roll(a, (-dy, -dx), axis=(0, 1))


def fused_response(img, k=0.06, sigma_d=1.0, sigma_i=2.5, grad=0):
    """R of the fused kernel (fp32), its trace plane, valid away from the border (crop >= 12 pixels)."""
    wd = taps(sigma_d).astype(F)
    wi = taps(sigma_i).astype(F)
    gscale = F(1.0) if grad == 1 else F(0.25)
    wir = (gscale * wi).astype(F)
    RD, RI = len(wd) - 1, len(wi) - 1
    v = img.astype(F)
    # stage B: acc = w0*v; acc = fma(w_t, v[-t] + v[+t], acc)
    acc = (wd[0] * v).astype(F)
    for t in range(1, RD + 1):
        acc = fma((shift(v, 0, -t) + shift(v, 0, t)).astype(F), wd[t], acc)
    T = acc
    # stage C: acc = 0; ascending rows: acc = fma(w|t|, T[row], acc)
    acc = np.zeros_like(T)
    for t in range(-RD, RD + 1):
        acc = fma(shift(T, t, 0), wd[abs(t)], acc)
    Is = acc
    # stage D: gradient, products, row blur (ascending x)
    if grad == 0:
        gx = (shift(Is, 0, 1) - shift(Is, 0, -1)).astype(F)
        gy = (shift(Is, 1, 0) - shift(Is, -1, 0)).astype(F)
    else:
        d = (shift(Is, -1, 1) + shift(Is, 1, 1) - shift(Is, -1, -1) - shift(Is, 1, -1)).astype(F)
        gx = fma((shift(Is, 0, 1) - shift(Is, 0, -1)).astype(F), F(0.25), (F(0.125) * d).astype(F))
        d = (shift(Is, 1, 1) + shift(Is, 1, -1) - shift(Is, -1, 1) - shift(Is, -1, -1)).astype(F)
        gy = fma((shift(Is, 1, 0) - shift(Is, -1, 0)).astype(F), F(0.25), (F(0.125) * d).astype(F))
    planes = [(gx * gx).astype(F), (gx * gy).astype(F), (gy * gy).astype(F)]
    out = []
    for p in planes:
        acc = np.zeros_like(p)
        for t in range(-RI, RI + 1):
            acc = fma(shift(p, 0, t), wir[abs(t)], acc)
        row = acc
        acc = np.zeros_like(p)
        for t in range(-RI, RI + 1):
            acc = fma(shift(row, t, 0), wi[abs(t)], acc)
        out.append(acc)
    A, B, C = out
    det = ((A * C).astype(F) - (B * B).astype(F)).astype(F)
    tr = (A + C).astype(F)
    R = (det - ((F(k) * tr).astype(F) * tr).astype(F)).astype(F)
    return R, tr


def eps(T, M, k=0.06):
    """harris_eps of harris_kernels3.cuh, same float operations."""
    T = np.asarray(T, F)
    M = np.asarray(M, F)
    eI = (F(17.0) * U * M).astype(F)
    eT = (F(2.0) * eI * np.sqrt(T).astype(F) + (eI * eI + F(64.0) * U * T)).astype(F)
    kk = F(abs(k))
    e = ((F(2.0) + F(4.0) * kk) * (T * eT + eT * eT) + F(2.0) * (F(1.0) + F(3.0) * kk) * U * T * T).astype(F)
    return (e * F(1.25) + F(1e-30)).astype(F)


def trace_cut(Th):
    """harris_trace_cut of harris_kernels3.cuh (u8 frames, Harris measure, k >= 0), same float operations."""
    if not Th > 0:
        return F(0)
    cut = F(2.0) * np.sqrt(F(Th)).astype(F) * (F(1.0) - F(1e-6)) - F(2.0) * F(0.2172) * F(1.25)
    return cut if cut > 0 else F(0)
