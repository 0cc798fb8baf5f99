/* Support routines for the generated PH-LAB plant right-hand side (device build; the oracle keeps its own copy:
 * reference native plant = /root/reference/envs/<variant>/_citation*.so).  Semantics follow the
 * reference binary's helpers:
 *   plant_index   <- rt_GetLookupIndex  (_citation.so @0xf470; SURVEY.md A.1)
 *   plant_table3  <- table3 S-function mdlOutputs/Table2 (@0x10da0 / @0x10a30)
 *   plant_powd_snf<- rt_powd_snf (@0x5d40)
 * Shared between the host oracle build (gcc, fp64, -ffp-contract=off) and the device build (nvcc). */
#ifndef PLANT_SUPPORT_H
#define PLANT_SUPPORT_H

#ifndef PLANT_FN
#define PLANT_FN static inline
#endif

/* breakpoint search: 0 if u <= x[0]; n-2 if u >= x[n-1]; else bisection with the reference's tie rule
 * (u >= 0: x[i] < u <= x[i+1];  u < 0: x[i] <= u < x[i+1]). */
PLANT_FN int plant_index(const real* x, int n, real u)
{
    if (x[0] >= u) return 0;
    if (!(u < x[n - 1])) return n - 2;
    int bottom = 0, top = n - 1;
    if (u >= (real)0) {
        for (;;) {
            int idx = (bottom + top) / 2;
            if (x[idx] < u) {
                bottom = idx + 1;
                if (u > x[bottom]) continue;
                return idx;
            }
            top = idx - 1;
        }
    } else {
        for (;;) {
            int idx = (bottom + top) / 2;
            if (x[idx] <= u) {
                bottom = idx + 1;
                if (u < x[bottom]) return idx;
                continue;
            }
            top = idx - 1;
        }
    }
}

/* bucketed breakpoint search (tools/lift/bucket.py), the counted search #{1 <= j <= n-2 : x[j] < y} in O(1): the uniform
 * cell floor(fma(y, s, o)), clamped to [0, nb - 1] (NaN -> 0), holds at most the one breakpoint x[n0 + 1], and its byte in
 * bkt (PLANT_BKT: plant_bucket_blob, staged next to the tables) is n0.  The generator emits it only where it has proved the
 * result equal to the counted search for every double and NaN.  A search with negative breakpoints (tie rule `x[j] <= u`
 * for those) passes y = plant_tie_up(u): b <= u  <=>  b < (the next double above u) for u < 0. */
#ifdef __CUDACC__
PLANT_FN int plant_cell(double v, int nb) { return min(max(__double2int_rd(v), 0), nb - 1); }       /* NaN converts to 0 */
PLANT_FN double plant_tie_up(double u) { return u < 0.0 ? __longlong_as_double(__double_as_longlong(u) - 1) : u; }
#else
PLANT_FN int plant_cell(double v, int nb) { return v >= 1.0 ? (v < (double)(nb - 1) ? (int)v : nb - 1) : 0; }
PLANT_FN double plant_tie_up(double u)
{
    union { double d; long long i; } b;
    b.d = u;
    b.i -= 1;
    return u < 0.0 ? b.d : u;
}
#endif
PLANT_FN int plant_bucket(double y, double s, double o, int nb, const unsigned char* bkt, const real* x)
{
    const int n0 = bkt[plant_cell(fma(y, s, o), nb)];
    return n0 + (x[n0 + 1] < y);
}

/* interval of the table3 S-function: the first breakpoint not below u, minus one, clamped to [0, n-2].  Breakpoints are
 * strictly increasing, so "scan while x[i] < u" stops after exactly count(x[i] < u) steps: written as that count, the search
 * has no data-dependent loop (n is a literal at every call, the sum unrolls into compare + add). */
PLANT_FN int plant_t3_interval(const real* x, int n, real u)
{
    int i = -1;
    for (int j = 0; j < n; ++j) i += (x[j] < u) ? 1 : 0;
    if (i < 0) i = 0;
    if (i > n - 2) i = n - 2;
    return i;
}

#ifndef PLANT_T3_DIV
#define PLANT_T3_DIV(a, b) ((a) / (b))
#endif
PLANT_FN real plant_t3_lerp(real v0, real v1, real u, real xlo, real xhi)
{
    const real y = PLANT_T3_DIV((v1 - v0) * (u - xlo), (xhi - xlo)) + v0;
    return (u == xhi) ? v1 : y;
}

PLANT_FN real plant_table3(const real* P1, int n1, const real* P2, int n2, const real* P3, int n3,
                           const real* P4, real u0, real u1, real u2)
{
    const int i1 = plant_t3_interval(P1, n1, u0);
    const int i2 = plant_t3_interval(P2, n2, u1);
    const int i3 = plant_t3_interval(P3, n3, u2);
    real t[2];
    for (int k = 0; k < 2; ++k) {
        const real* slab = P4 + (i3 + k) * n1 * n2;
        real w[2];
        for (int j = 0; j < 2; ++j) {
            const real v0 = slab[i1 * n2 + i2 + j];
            const real v1 = slab[(i1 + 1) * n2 + i2 + j];
            w[j] = plant_t3_lerp(v0, v1, u0, P1[i1], P1[i1 + 1]);
        }
        t[k] = plant_t3_lerp(w[0], w[1], u1, P2[i2], P2[i2 + 1]);
    }
    return plant_t3_lerp(t[0], t[1], u2, P3[i3], P3[i3 + 1]);
}

#endif
