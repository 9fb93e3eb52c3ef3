/* detmath.h -- deterministic double-precision sin / cos / atan2 in plain IEEE-754 arithmetic (+, -, *, / only; no FMA,
 * no library calls), so that a host build (-ffp-contract=off) and a device build (-fmad=false) return bit-identical
 * results.  The line front end (LSD region angles, rectangle axes, KeyLine::angle, LBD line direction) calls
 * cos/sin/atan2 of the platform's libm in the reference (LSDDetector_custom.cpp:290, binary_descriptor_custom.cpp:
 * 1119-1120 and OpenCV's lsd.cpp); libm results are not portable to the GPU, so the determinism rule of this
 * restatement is "evaluate with these kernels in double, then round to the type the reference stores".
 *
 * Argument reduction: Cody-Waite with a 3-part pi/2 (valid for |x| < ~1e5, far above the [-4 pi, 4 pi] needed here);
 * kernels: the classical minimax polynomials on [-pi/4, pi/4] (sin: degree 13, cos: degree 14) and the 4-interval
 * arctangent with an odd degree-23 polynomial.  Measured against glibc: max |err| < 2.3e-16 (tests/test_lines_oracle.py).
 *
 * The library (nvcc -fmad=false), the oracle (g++ -ffp-contract=off) and the CPU emulators of tests/cta_emu compile
 * this one text, so the device and the oracle evaluate the same expressions.
 */
#ifndef PLP_DETMATH_H
#define PLP_DETMATH_H

#if defined(__CUDACC__)
#define DET_HD __host__ __device__ __forceinline__
#else
#define DET_HD static inline
#endif

DET_HD double det_kernel_sin(double x) {
    const double S1 = -1.66666666666666324348e-01, S2 = 8.33333333332248946124e-03, S3 = -1.98412698298579493134e-04,
                 S4 = 2.75573137070700676789e-06, S5 = -2.50507602534068634195e-08, S6 = 1.58969099521155010221e-10;
    const double z = x * x;
    const double r = S2 + z * (S3 + z * (S4 + z * (S5 + z * S6)));
    return x + (z * x) * (S1 + z * r);
}

DET_HD double det_kernel_cos(double x) {
    const double C1 = 4.16666666666666019037e-02, C2 = -1.38888888888741095749e-03, C3 = 2.48015872894767294178e-05,
                 C4 = -2.75573143513906633035e-07, C5 = 2.08757232129817482790e-09, C6 = -1.13596475577881948265e-11;
    const double z = x * x;
    const double r = z * (C1 + z * (C2 + z * (C3 + z * (C4 + z * (C5 + z * C6)))));
    const double hz = 0.5 * z;
    const double w = 1.0 - hz;
    return w + (((1.0 - w) - hz) + z * r);
}

/* x = n * pi/2 + r, |r| <= pi/4 (+ rounding); returns n mod 4 */
DET_HD int det_rem_pio2(double x, double *r) {
    const double INV_PIO2 = 6.36619772367581382433e-01;
    const double P1 = 1.57079632673412561417e+00; /* first 33 bits of pi/2 */
    const double P2 = 6.07710050630396597660e-11; /* next 33 bits */
    const double P3 = 2.02226624879595063154e-21; /* the rest */
    const double t = x * INV_PIO2;
    const double fn = (double)(long long)(t + (t >= 0.0 ? 0.5 : -0.5));
    double y = x - fn * P1;
    y = y - fn * P2;
    y = y - fn * P3;
    *r = y;
    return (int)(((long long)fn) & 3);
}

DET_HD double det_sin(double x) {
    double r;
    const int n = det_rem_pio2(x, &r);
    switch (n) {
        case 0: return det_kernel_sin(r);
        case 1: return det_kernel_cos(r);
        case 2: return -det_kernel_sin(r);
        default: return -det_kernel_cos(r);
    }
}

DET_HD double det_cos(double x) {
    double r;
    const int n = det_rem_pio2(x, &r);
    switch (n) {
        case 0: return det_kernel_cos(r);
        case 1: return -det_kernel_sin(r);
        case 2: return -det_kernel_cos(r);
        default: return det_kernel_sin(r);
    }
}

DET_HD double det_atan_pos(double x) { /* x >= 0 */
    const double aT0 = 3.33333333333329318027e-01, aT1 = -1.99999999998764832476e-01, aT2 = 1.42857142725034663711e-01,
                 aT3 = -1.11111104054623557880e-01, aT4 = 9.09088713343650656196e-02, aT5 = -7.69187620504482999495e-02,
                 aT6 = 6.66107313738753120669e-02, aT7 = -5.83357013379057348645e-02, aT8 = 4.97687799461593236017e-02,
                 aT9 = -3.65315727442169155270e-02, aT10 = 1.62858201153657823623e-02;
    double hi, lo, t;
    int id;
    if (x < 0.4375) {
        id = -1; t = x; hi = 0.0; lo = 0.0;
    } else if (x < 0.6875) {
        id = 0; t = (2.0 * x - 1.0) / (2.0 + x);
        hi = 4.63647609000806093515e-01; lo = 2.26987774529616870924e-17;
    } else if (x < 1.1875) {
        id = 1; t = (x - 1.0) / (x + 1.0);
        hi = 7.85398163397448278999e-01; lo = 3.06161699786838301793e-17;
    } else if (x < 2.4375) {
        id = 2; t = (x - 1.5) / (1.0 + 1.5 * x);
        hi = 9.82793723247329054082e-01; lo = 1.39033110312309984516e-17;
    } else {
        id = 3; t = -1.0 / x;
        hi = 1.57079632679489655800e+00; lo = 6.12323399573676603587e-17;
    }
    const double z = t * t;
    const double w = z * z;
    const double s1 = z * (aT0 + w * (aT2 + w * (aT4 + w * (aT6 + w * (aT8 + w * aT10)))));
    const double s2 = w * (aT1 + w * (aT3 + w * (aT5 + w * (aT7 + w * aT9))));
    if (id < 0) return t - t * (s1 + s2);
    return hi - ((t * (s1 + s2) - lo) - t);
}

DET_HD double det_atan2(double y, double x) {
    const double PI = 3.14159265358979311600e+00, PI_LO = 1.22464679914735317720e-16;
    if (x == 0.0 && y == 0.0) return 0.0;
    const double ay = y < 0.0 ? -y : y, ax = x < 0.0 ? -x : x;
    double a;
    if (ax == 0.0) a = 1.57079632679489655800e+00;
    else a = det_atan_pos(ay / ax);
    if (x < 0.0) a = PI - (a - PI_LO);
    return y < 0.0 ? -a : a;
}

#endif
