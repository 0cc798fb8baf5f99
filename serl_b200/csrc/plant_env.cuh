// Device code shared by the rollout kernels (rollout.cu: K1 warp-GEMV actor; rollout_tc.cu: wgmma actor for wide
// two-hidden-layer policies): the generated PH-LAB plant, the ode5 step, CitationEnv (reset / step / reward / termination,
// envs/phlabenv.py:401-482), the launch argument block, and the mbarrier / TMA primitives.  Every translation unit that
// includes this file gets its own copy of the (static) tables and __noinline__ plant functions.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/serl_b200.h"
#include "common.cuh"
#include "actor_math.cuh"

#ifdef PLANT_F32
typedef float real;      // experimental build: single-precision right-hand side, double-precision integrator state
#else
typedef double real;
#endif
// lookup tables: one blob (gen/plant_tables_blob.h) that the kernels stage into shared memory; the generated
// right-hand sides address it through the `plant_tab` pointer they are handed.
#define PLANT_TAB(name) (plant_tab + PT_OFF_##name)
#define PLANT_XARGS , const real* __restrict__ plant_tab
// ---- fast fp64 math for the device plant (<= ~1 ulp; the oracle keeps the reference's exact operations) -------
// division: 20-bit hardware reciprocal seed + two Newton steps + one residual correction (9 instructions instead of ~33)
__device__ __forceinline__ double plant_div_fast(double a, double b)
{
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(b));
    double e = fma(-b, r, 1.0);
    r = fma(r, e, r);
    e = fma(-b, r, 1.0);
    r = fma(r, e, r);
    const double q = a * r;
    return fma(fma(-b, q, a), r, q);
}
// sqrt: 20-bit rsqrt seed + two Newton steps + residual correction, WITHOUT a branch: the right-hand side evaluates
// signed square roots as sqrt(-x), sqrt(x) + select, so one argument of each pair is negative at every call, and a
// fallback branch to the library would be taken four times per evaluation (and would cut the function into basic blocks
// the scheduler cannot move work across).  Special cases by select: negative / NaN -> NaN (the seed already is),
// 0 and denormals -> 0 (the seed flushes them to zero), +inf -> +inf.
__device__ __forceinline__ double plant_sqrt_fast(double x)
{
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    const double hx = 0.5 * x;
    y = y * fma(-hx * y, y, 1.5);
    y = y * fma(-hx * y, y, 1.5);
    const double s = x * y;
    double r = fma(fma(-s, s, x), 0.5 * y, s);
    r = (x >= 0.0 && x < 2.2250738585072014e-308) ? 0.0 : r;
    r = (x == __longlong_as_double(0x7ff0000000000000ll)) ? x : r;
    return r;
}
// sincos: two-term Cody-Waite reduction by pi/2 (106 bits of pi/2: accurate to ~1 ulp far beyond the angles a flying
// aircraft can reach; episodes end when an attitude limit trips) and the fdlibm kernel polynomials, no branch.  |x| > 2^20
// (a diverged state; NaN likewise) returns NaN, which the rollout kernels report through the status word.
__device__ __forceinline__ void plant_sincos_fast(double x, double* sp, double* cp)
{
    const double q = rint(x * 0.6366197723675814);
    double r = fma(-q, 1.5707963267948966, x);
    r = fma(-q, 6.123233995736766e-17, r);
    r = (fabs(x) <= 1048576.0) ? r : __longlong_as_double(0x7ff8000000000000ll);
    const double z = r * r;
    double ps = 1.58969099521155010221e-10;
    ps = fma(ps, z, -2.50507602534068634195e-08);
    ps = fma(ps, z, 2.75573137070700676789e-06);
    ps = fma(ps, z, -1.98412698298579493134e-04);
    ps = fma(ps, z, 8.33333333332248946124e-03);
    ps = fma(ps, z, -1.66666666666666324348e-01);
    const double s = fma(r * z, ps, r);
    double pc = -1.13596475577881948265e-11;
    pc = fma(pc, z, 2.08757232129817482790e-09);
    pc = fma(pc, z, -2.75573143513906633035e-07);
    pc = fma(pc, z, 2.48015872894767294178e-05);
    pc = fma(pc, z, -1.38888888888741095749e-03);
    pc = fma(pc, z, 4.16666666666666019037e-02);
    const double c = fma(z * z, pc, fma(-0.5, z, 1.0));
    const int n = (int)q & 3;
    const double s1 = (n & 1) ? c : s, c1 = (n & 1) ? s : c;
    *sp = (n & 2) ? -s1 : s1;
    *cp = ((n + 1) & 2) ? -c1 : c1;
}
// log / exp / pow for the atmosphere model (density ~ (T / T0)^4.26; exp only above 11 km): the fdlibm kernels (e_log.c,
// e_exp.c) without their special-case branches, divisions by plant_div_fast.  log, exp <= 1 ulp; pow = exp(b log a) carries
// the rounding of b log a: <= (2 + |b ln a|) ulp, i.e. <= 3.5 ulp for the temperature ratios of 0 - 11 km.  a <= 0, NaN
// or inf returns NaN (-> status word of the rollout kernels).
__device__ __forceinline__ double plant_log_fast(double a)
{
    const long long ia = __double_as_longlong(a);
    const long long top = (ia >> 32) + (0x3ff00000 - 0x3fe6a09e);           // a = 2^k * m, m in [sqrt(2)/2, sqrt(2))
    const int k = (int)(top >> 20) - 0x3ff;
    const long long hm = (top & 0x000fffff) + 0x3fe6a09e;
    const double m = __longlong_as_double((hm << 32) | (ia & 0xffffffffll));
    const double f = m - 1.0;
    const double s = plant_div_fast(f, 2.0 + f);
    const double z = s * s, w = z * z;
    const double t1 = w * fma(w, fma(w, 1.531383769920937332e-01, 2.222219843214978396e-01), 3.999999999940941908e-01);
    const double t2 = z * fma(w, fma(w, fma(w, 1.479819860511658591e-01, 1.818357216161805012e-01), 2.857142874366239149e-01),
                              6.666666666666735130e-01);
    const double R = t2 + t1;
    const double hfsq = 0.5 * f * f;
    const double dk = (double)k;
    return dk * 6.93147180369123816490e-01 - ((hfsq - fma(s, hfsq + R, dk * 1.90821492927058770002e-10)) - f);
}
__device__ __forceinline__ double plant_exp_fast(double x)          // |x| < 700
{
    const double kd = rint(x * 1.44269504088896338700e+00);
    const double hi = fma(-kd, 6.93147180369123816490e-01, x);
    const double lo = kd * 1.90821492927058770002e-10;
    const double r = hi - lo;
    const double t = r * r;
    const double c = r - t * fma(t, fma(t, fma(t, fma(t, 4.13813679705723846039e-08, -1.65339022054652515390e-06),
                                               6.61375632143793436117e-05), -2.77777777770155933842e-03), 1.66666666666666019037e-01);
    const double y = 1.0 - ((lo - plant_div_fast(r * c, 2.0 - c)) - hi);
    return __longlong_as_double(__double_as_longlong(y) + ((long long)(int)kd << 52));
}
__device__ __forceinline__ double plant_pow_fast(double a, double b)
{
    const double y = plant_exp_fast(b * plant_log_fast(a));
    return (a > 0.0 && a < 1e300) ? y : __longlong_as_double(0x7ff8000000000000ll);
}
__device__ __forceinline__ double plant_sin_fast(double x) { double s, c; plant_sincos_fast(x, &s, &c); return s; }
__device__ __forceinline__ double plant_cos_fast(double x) { double s, c; plant_sincos_fast(x, &s, &c); return c; }
#if defined(PLANT_F32)
// experimental build (`python -m serl_b200.build --f32`): fp32 right-hand side (BASELINE north_star: "fp32 ODE integration")
#define PLANT_GEN(f) PLANT_STR(gen_f32/f)
#define PLANT_DIV(a, b) ((a) / (b))
#define PLANT_SQRT sqrtf
#define PLANT_FABS fabsf
#define PLANT_SIN sinf
#define PLANT_COS cosf
#define PLANT_SINCOS sincosf
#define PLANT_TAN tanf
#define PLANT_EXP expf
#define PLANT_LOG10 log10f
#define PLANT_POW powf
#elif defined(PLANT_EXACT)
// validation build (`python -m serl_b200.build --exact`): reference operation order, library math, no FMA contraction
#define PLANT_GEN(f) PLANT_STR(gen_exact/f)
#define PLANT_DIV(a, b) ((a) / (b))
#define PLANT_SQRT sqrt
#define PLANT_FABS fabs
#define PLANT_SIN sin
#define PLANT_COS cos
#define PLANT_SINCOS sincos
#else
#define PLANT_GEN(f) PLANT_STR(gen/f)
#define PLANT_DIV(a, b) plant_div_fast((a), (b))
#define PLANT_T3_DIV(a, b) plant_div_fast((a), (b))
#define PLANT_SQRT plant_sqrt_fast
#define PLANT_FABS fabs
#define PLANT_SIN plant_sin_fast
#define PLANT_COS plant_cos_fast
#define PLANT_SINCOS plant_sincos_fast
#endif
#ifndef PLANT_F32
#define PLANT_TAN tan
#define PLANT_LOG10 log10
#ifdef PLANT_EXACT
#define PLANT_EXP exp
#define PLANT_POW pow
#else
#define PLANT_EXP plant_exp_fast
#define PLANT_POW plant_pow_fast
#endif
#endif
#define PLANT_STR(x) #x
#define PLANT_FN static __device__ __forceinline__
#include "plant_support.h"
#undef PLANT_FN
#define PLANT_FN static __device__ __noinline__
#include PLANT_GEN(plant_tables_blob.h)
#define PLANT_CONSTS(n) static __constant__ real plant_k[n]
#define PLANT_K(i) plant_k[i]
#include PLANT_GEN(plant_consts.h)
#define PLANT_IC(v) static __device__ const double plant_ic_unused_##v[19]
#define PLANT_IC_TABLE static __device__ const double plant_ic_table[SERL_PLANT_COUNT][19]
#define PLANT_PV_TABLE static __device__ const real plant_pv[SERL_PLANT_COUNT][PLANT_NPV]
#define PLANT_PV(k) plant_pvrow[k]
// the right-hand side works on the 14 live continuous states only: rtX index -> position in the compact arrays
#define PLANT_XI(i) ((i) < 8 ? (i) : ((i) == 9 ? 8 : ((i) == 12 ? 9 : (i) - 5)))
#include PLANT_GEN(plant_ic.h)
// The generated right-hand sides are inlined into the by-value wrappers plant_rhs_regs / plant_rhs_regs_smem below.
#undef PLANT_FN
#define PLANT_FN static __device__ __forceinline__
#define PLANT_RHS_COMMON_NAME plant_rhs_common
// Breakpoint searches: the counted form here (tables through a generic pointer: the bucketed form's two dependent table
// reads cost more than its compares save); the bucketed one (tools/lift/bucket.py) in the shared-space instance below when
// the including kernel stages the byte tables (PLANT_SMEM_BUCKETS)
#undef PLANT_SEARCH
#define PLANT_SEARCH(bucketed, counted) (counted)
#include PLANT_GEN(plant_rhs_common.h)     // ONE function for every plant variant + per-variant parameter rows
// Second instance of the same generated text for kernels that stage the tables (+ parameter rows) at the START of their
// dynamic shared memory: tables and parameter rows are read as plant_smem_tab[...] — the compiler sees the shared address
// space and emits LDS with 32-bit immediate-offset addressing.  Through the generic `plant_tab` pointer of the first
// instance every one of the ~220 table reads of a right-hand side cost a 64-bit address computation (IADD3 pairs), an
// R2UR of the base pointer and a generic LD: ~11 % of the function's instructions.
// Every kernel that uses the shared-space instance declares its dynamic shared memory with the SAME alignment as this
// symbol (128): nvcc places each `extern __shared__` array at (end of the kernel's static shared memory) rounded up to that
// array's own alignment, so differently aligned declarations can name different addresses (plant_tab_check() traps then).
extern __shared__ __align__(128) real plant_smem_tab[];
__device__ __forceinline__ void plant_tab_check(const void* dynamic_smem_base)
{
    if ((const void*)plant_smem_tab != dynamic_smem_base) __trap();
}
__device__ __forceinline__ int plant_smem_index(const real* p)          // element index of a generic pointer into the staged blob
{
    return (int)((unsigned)__cvta_generic_to_shared(p) - (unsigned)__cvta_generic_to_shared(plant_smem_tab)) / (int)sizeof(real);
}
#undef PLANT_TAB
#undef PLANT_PV
#undef PLANT_PV_TABLE
#define PLANT_TAB(name) (plant_smem_tab + PT_OFF_##name)
#define PLANT_PV(k) plant_smem_tab[plant_smem_index(plant_pvrow) + (k)]
#define PLANT_PV_TABLE static __device__ const real plant_pv_second_instance_unused[SERL_PLANT_COUNT][PLANT_NPV]
#undef PLANT_RHS_COMMON_NAME
#define PLANT_RHS_COMMON_NAME plant_rhs_common_smem
#if defined(PLANT_SMEM_BUCKETS) && defined(PLANT_BUCKET_BYTES)
// the byte tables of the bucketed searches follow the parameter rows (plant_stage_buckets)
#undef PLANT_SEARCH
#define PLANT_SEARCH(bucketed, counted) (bucketed)
#define PLANT_BKT(name) (reinterpret_cast<const unsigned char*>(plant_smem_tab + PT_TOTAL + SERL_PLANT_COUNT * PLANT_NPV) + PB_OFF_##name)
#endif
#include PLANT_GEN(plant_rhs_common.h)
#undef PLANT_SEARCH
#define PLANT_SEARCH(bucketed, counted) (counted)
#undef PLANT_BKT
#undef PLANT_RHS_COMMON_NAME
#undef PLANT_TAB
#undef PLANT_PV
#undef PLANT_FN
#define PLANT_FN static __device__ __noinline__
#define PLANT_TAB(name) (plant_tab + PT_OFF_##name)
#define PLANT_PV(k) plant_pvrow[k]
#undef PLANT_XI
#define PLANT_XI(i) (i)                    // trace-only navigation states: full rtX indexing
#include PLANT_GEN(plant_rhs_nav.h)


#define NX 19
#define NLIVE 14
#define MAX_CTA_THREADS 256

// State vectors travel BY VALUE between the out-of-line plant functions: the struct arguments and results of a
// __noinline__ function are passed in registers, whereas an array whose address is handed to one lives in local memory
// (an L2 round trip inside the stage-to-stage dependency chain of the integrator).
struct PlantLive { real v[NLIVE]; };       // live continuous states / their derivatives, compact order (PLANT_XI)
struct PlantState { double v[NX]; };       // the integrator state rtX
// ONE out-of-line copy of the right-hand side per table address space (the generated body is inlined here only)
static __device__ __noinline__ PlantLive plant_rhs_regs(PlantLive x, real u0, real u1, real u2, real u3, const real* tab,
                                                        const real* pvrow)
{
    const real u[4] = {u0, u1, u2, u3};
    PlantLive d;
    plant_rhs_common(x.v, u, d.v, tab, pvrow);
    return d;
}
static __device__ __noinline__ PlantLive plant_rhs_regs_smem(PlantLive x, real u0, real u1, real u2, real u3, const real* tab,
                                                             const real* pvrow)
{
    const real u[4] = {u0, u1, u2, u3};
    PlantLive d;
    plant_rhs_common_smem(x.v, u, d.v, tab, pvrow);
    return d;
}

// live continuous states of the plant (SURVEY.md 2.3): p q r V alpha beta phi theta | h | washout | N1 N1 N2 N2
// (psi, x_e, y_e never feed back and are integrated only for traces; Parameter_CSTATE(_g) are folded constants).
// `pv` = this variant's parameter row (shared memory copy of plant_pv, or the global table).

__device__ __forceinline__ const double* plant_ic(int variant) { return plant_ic_table[variant]; }

// Simulink fixed-step ode5 exactly as inlined in the reference's step(): stage states are
// y + (f0*hB0 + f1*hB1 + ...) with hB = h*B[s][j], summed left to right (zero coefficients included).
#define ODE5_B_INIT { \
        {1.0 / 5.0, 0, 0, 0, 0, 0}, \
        {3.0 / 40.0, 9.0 / 40.0, 0, 0, 0, 0}, \
        {44.0 / 45.0, -56.0 / 15.0, 32.0 / 9.0, 0, 0, 0}, \
        {19372.0 / 6561.0, -25360.0 / 2187.0, 64448.0 / 6561.0, -212.0 / 729.0, 0, 0}, \
        {9017.0 / 3168.0, -355.0 / 33.0, 46732.0 / 5247.0, 49.0 / 176.0, -5103.0 / 18656.0, 0}, \
        {35.0 / 384.0, 0, 500.0 / 1113.0, 125.0 / 192.0, -2187.0 / 6784.0, 11.0 / 84.0}}
#define ODE5_LIVE_INIT {0, 1, 2, 3, 4, 5, 6, 7, 9, 12, 15, 16, 17, 18}
static __constant__ double c_ode5_B[6][6] = ODE5_B_INIT;      // dynamically indexed copy (trace path)
static __constant__ int c_ode5_live[NLIVE] = ODE5_LIVE_INIT;

// trace mode only: psi, x_e, y_e (rtX 8, 10, 11).  Their derivatives depend on the live states alone, so they are
// integrated after the fact with the same stage states, rebuilt from the stored stage derivatives f[6][NLIVE].
static __device__ __noinline__ void plant_step_nav(double* Xnav, const double* X0, const real (*f)[NLIVE], const real* U, const real* tab)
{
    const double h = 0.01;
    const int NAV[3] = {8, 10, 11};
    double g[6][3], xs[NX];
    real xr[NX], xd[NX];
#pragma unroll 1
    for (int s = 0; s < 6; ++s) {
        for (int i = 0; i < NX; ++i) xs[i] = X0[i];
        if (s > 0) {
            for (int li = 0; li < NLIVE; ++li) {
                const int i = c_ode5_live[li];
                double acc = (double)f[0][li] * (h * c_ode5_B[s - 1][0]);
                for (int j = 1; j < s; ++j) acc += (double)f[j][li] * (h * c_ode5_B[s - 1][j]);
                xs[i] = X0[i] + acc;
            }
            for (int q = 0; q < 3; ++q) {
                double acc = g[0][q] * (h * c_ode5_B[s - 1][0]);
                for (int j = 1; j < s; ++j) acc += g[j][q] * (h * c_ode5_B[s - 1][j]);
                xs[NAV[q]] = X0[NAV[q]] + acc;
            }
        }
        for (int i = 0; i < NX; ++i) xr[i] = (real)xs[i];
        plant_rhs_nav(xr, U, xd, tab);
        g[s][0] = (double)xd[8]; g[s][1] = (double)xd[10]; g[s][2] = (double)xd[11];
    }
    for (int q = 0; q < 3; ++q) {
        double acc = g[0][q] * (h * c_ode5_B[5][0]);
        for (int j = 1; j < 6; ++j) acc += g[j][q] * (h * c_ode5_B[5][j]);
        Xnav[q] = X0[NAV[q]] + acc;
    }
}

// Stage loop fully unrolled (h*B folds to constants).  The right-hand side is ONE __noinline__ function (the same code for
// every plant variant) that takes the stage state and returns the stage derivative by value.  The six stage derivatives
// (84 values, all live for the last combination) do not fit next to the rest in 255 registers: ptxas keeps part of them
// in local memory.  The integrator state and the
// stage combinations are double in every build; `real` (the type of the right-hand side) is double unless PLANT_F32.
// pv_post / call: time-triggered builds (cg_timed): the parameter row switches to pv_post when the model clock
// call * 0.01 + c_s * 0.01 of a stage reaches 20 s: every stage from call SERL_TRIGGER_CALLS on, and the LAST stage (c = 1) of
// call SERL_TRIGGER_CALLS - 1, whose time 19.99 + 0.01 already compares >= 20 in the binary.
// STAB: tables + parameter rows staged at the start of dynamic shared memory (see plant_rhs_common_smem).
// GUST instantiation (launches with a `gust` env, SERL_MODE_GUST): bit 30 of `call` marks a gust env, and u[3], the
// right-hand side's angle-of-attack offset, is atan(w_gust / V) for the stages whose time lies in the pulse 20 s <= t <= 23 s
// (include/serl_b200.h).  Without GUST the offset is the constant 0 and the code is that of a build without the feature.
#define PLANT_CALL_GUST (1 << 30)
#define PLANT_CALL_GUST_UP (1 << 29)       // the `test` build: the same pulse with the opposite sign
__device__ __forceinline__ real plant_gust_offset(int call, int s, real V)
{
    const bool on = (call == SERL_TRIGGER_CALLS - 1 && s == 5) || (call >= SERL_TRIGGER_CALLS && call < SERL_GUST_END_CALLS) ||
                    (call == SERL_GUST_END_CALLS && s == 0);
    if (!on) return (real)0;
    return (real)(atan(PLANT_DIV((double)SERL_GUST_W, (double)V)) * 1.0);
}
// X (the state) and the command arrive by value and the new state is returned: nothing of the hot path has its address
// taken (see PlantState).  Only the trace path (nav) copies the stage derivatives to an array for plant_step_nav.
template <bool STAB = false, bool GUST = false>
static __device__ __noinline__ PlantState plant_step(const real* pv, PlantState X, double U0, double U1, double U2, const real* tab,
                                                     bool nav = false, const real* pv_post = nullptr, int call = 0)
{
    const bool gust = GUST && (call & PLANT_CALL_GUST) != 0, gust_up = GUST && (call & PLANT_CALL_GUST_UP) != 0;
    if (GUST) call &= ~(PLANT_CALL_GUST | PLANT_CALL_GUST_UP);
    constexpr double h = 0.01;
    constexpr double B[6][6] = ODE5_B_INIT;
    constexpr int LIVE[NLIVE] = ODE5_LIVE_INIT;
    const real u0 = (real)U0, u1 = (real)U1, u2 = (real)U2;
    real u3 = (real)0;
    PlantLive x;
#pragma unroll
    for (int li = 0; li < NLIVE; ++li) x.v[li] = (real)X.v[LIVE[li]];
    double xl[NLIVE];
    PlantLive f[6];
#pragma unroll
    for (int s = 0; s < 6; ++s) {
        const bool post = pv_post != nullptr && (call >= SERL_TRIGGER_CALLS || (s == 5 && call == SERL_TRIGGER_CALLS - 1));
        if (GUST) { u3 = gust ? plant_gust_offset(call, s, x.v[3]) : (real)0; if (gust_up) u3 = -u3; }
        f[s] = STAB ? plant_rhs_regs_smem(x, u0, u1, u2, u3, tab, post ? pv_post : pv)
                    : plant_rhs_regs(x, u0, u1, u2, u3, tab, post ? pv_post : pv);
#pragma unroll
        for (int li = 0; li < NLIVE; ++li) {
            double acc = (double)f[0].v[li] * (h * B[s][0]);
#pragma unroll
            for (int j = 1; j <= s; ++j) acc += (double)f[j].v[li] * (h * B[s][j]);
            xl[li] = X.v[LIVE[li]] + acc;
            x.v[li] = (real)xl[li];
        }
    }
    if (nav) {
        double X0[NX], xn[3];
        real fa[6][NLIVE];
        const real u[4] = {u0, u1, u2, u3};
#pragma unroll
        for (int i = 0; i < NX; ++i) X0[i] = X.v[i];
#pragma unroll
        for (int s = 0; s < 6; ++s)
#pragma unroll
            for (int li = 0; li < NLIVE; ++li) fa[s][li] = f[s].v[li];
        plant_step_nav(xn, X0, fa, u, tab);
        X.v[8] = xn[0]; X.v[10] = xn[1]; X.v[11] = xn[2];
    }
#pragma unroll
    for (int li = 0; li < NLIVE; ++li) X.v[LIVE[li]] = xl[li];
    return X;
}

// activations: IEEE-only sequences of actor_math.cuh (bit-reproducible on a CPU; see oracle/plant/actor_kernel_order.c)
__device__ __forceinline__ float act_fn(int act, float x) { return am_act1(act, x); }

// reference-signal value in degrees (serl_b200/refsig.py; recovered shape of signals.RandomizedCosineStepSequence)
__device__ __forceinline__ double ref_deg(const double* __restrict__ lv, const double* __restrict__ st, double t, double offset, double smooth_w)
{
    int k = 0;
#pragma unroll
    for (int j = 1; j < SERL_REF_BLOCKS; ++j)
        if (t >= st[j]) k = j;
    if (k == 0) return offset + lv[0];
    const double x = (t - st[k]) / smooth_w;
    if (x >= 1.0) return offset + lv[k];
    return offset + (lv[k - 1] + (lv[k] - lv[k - 1]) * (0.5 * (1.0 - cos(3.141592653589793 * x))));
}

// ---- per-trajectory environment (CitationEnv restated for one thread) --------------------------------------
// hand-over record of a trajectory that is continued by another CTA slot (time-split schedule, see rollout_kernel_persist)
struct Handoff {
    double* X;      // [NX][n]
    double* t;      // [n]
    double* ret;    // [n]
    float* obs;     // [7][n]; incremental launches (INC): [10][n], followed by last_u [3][n] f64; symmetric (SYM): [2][n]
    int* k;         // [n]  executed steps | done << 30
    int* flag;      // [n / 32] one word per warp, 1 when the record is complete
    long long n;
};

struct RolloutArgs {
    const float* weights; int P; serl_actor_shape sh;
    const double* ref_levels; const double* ref_starts; const int* env_mode; int n_envs; int horizon;
    const float* action_noise;      // optional [pop, n_envs, horizon, 3 (1 with symmetric control)]: clipped exploration noise (agent.py:90-93)
    double* returns; int* steps; double* trace;   // trace optional [pop, n_envs, horizon, SERL_TRACE_COLS]
    float* actions;                 // optional [pop, n_envs, horizon, 3] fp32: commanded deflection last_u (smoothness metric)
    int pop;
    double t_max;                   // episode length [s] (envs/phlabenv.py:181; 80 in evaluation mode :295-301)
    double smooth_w;                // width of the raised-cosine reference transitions [s] (t_max // 6)
    const int* env_order;           // optional [n_envs]: lane slot -> env index
    float* replay; int replay_env;  // optional [pop, horizon, SERL_REPLAY_COLS] transitions of one env per actor
    int* status;                    // optional device status word
    int sm_limit;                   // > 0: CTAs of the persistent kernel (SMs) this launch may use
    const float* sensor_noise;      // optional [pop, n_envs, horizon + 1, 7] standard-normal draws of the sensor-noise shim
    // persistent schedule
    const float* wt;                // [pop][P4] genomes in the shared-memory layout (transposed matrices), 16-byte aligned rows
    int P4;                         // row stride of wt / smem slot size in floats (multiple of 4)
    int apc, wps;                   // genome slots per CTA, warps per slot
    int stagger;                    // apc == 2: slot 1 runs half a step behind slot 0 (rollout_kernel_persist)
    int n_chunks;                   // env chunks of wps*32 lanes per actor
    long long n_tasks;              // pop * n_chunks
    long long n_slots;              // gridDim.x * apc
    Handoff ho;
};

// plant tables + per-variant parameter rows (reals), and that count rounded up to an even one: the block K1 stages at the
// start of its dynamic shared memory, in front of the genome slots
constexpr int PLANT_TABN = PT_TOTAL + SERL_PLANT_COUNT * PLANT_NPV;
#if defined(PLANT_SMEM_BUCKETS) && defined(PLANT_BUCKET_BYTES)
constexpr int PLANT_BKT_WORDS = (PLANT_BUCKET_BYTES + 7) / 8;       // byte tables of the bucketed searches, in doubles
#else
constexpr int PLANT_BKT_WORDS = 0;
#endif
// a kernel that stages the tables: tables | parameter rows | byte tables of the bucketed searches (PLANT_SMEM_BUCKETS)
constexpr int PLANT_TABN2 = (PLANT_TABN + PLANT_BKT_WORDS + 1) & ~1;
__device__ __forceinline__ void plant_stage_buckets(real* tab_s, int tid, int nthreads)
{
#if defined(PLANT_SMEM_BUCKETS) && defined(PLANT_BUCKET_BYTES)
    unsigned char* b = reinterpret_cast<unsigned char*>(tab_s + PLANT_TABN);
    for (int i = tid; i < PLANT_BUCKET_BYTES; i += nthreads) b[i] = plant_bucket_blob[i];
#endif
}

// Tracking-error accumulators of the evaluation suite (serl_rollout_desc.d_track): the kernels take them as a launch
// argument of their own, next to the argument block, so that adding them moved no field of the training instantiations.
//   out  [pop * n_envs][SERL_TRACK_COLS] f64, written at the end of each trajectory
//   ho   [TRACK_CARRY][Handoff.n] f64: the sums, the carried controlled state and the cost tally of a trajectory K1's
//        time-split schedule hands to another slot (the rest of its record is Handoff)
//   cost optional [pop * n_envs] int32 (serl_rollout_desc.d_cost): executed steps whose cost flag is set
struct TrackArgs { double* out; double* ho; int* cost; };
#define TRACK_COST (SERL_TRACK_COLS + 3)      // Env::trk: steps with the cost flag set so far (an exact integer in f64)
#define TRACK_V0 (SERL_TRACK_COLS + 4)        // Env::trk: V0 of the env's plant variant, the airspeed bound of get_cost
#define TRACK_CARRY (SERL_TRACK_COLS + 5)

struct Env {
    double X[NX];
    const real* tab;         // plant tables (shared or global memory)
    const real* pv;          // parameter row of this env's plant variant
    const real* pv_post;     // row after the trigger of a time-triggered build, or nullptr
    const double* ref_lv;    // this env's reference-signal levels / starts [2][SERL_REF_BLOCKS] (global, read per step)
    const double* ref_st;
    double t, ret, theta_trim;
    int fault, k;
    bool done;
    int gust;                // env_mode >> 24: 1 = SERL_MODE_GUST, 3 = with SERL_MODE_GUST_UP
    // TRACK instantiations only: sum |e_theta|, sum |e_phi|, sum |e_beta|, sum e_beta, then the controlled state
    // (theta, phi, beta) of env.x when the next step starts, the cost tally and V0 (TRACK_COST, TRACK_V0)
    double trk[TRACK_CARRY];
};

// one plant step of the env (reset's zero-command step and env_step share this single plant_step instance)
template <bool STAB, bool GUST>
__device__ __forceinline__ void plant_step_env(Env& e, const double* cmd, bool nav, int call)
{
    PlantState s;
#pragma unroll
    for (int i = 0; i < NX; ++i) s.v[i] = e.X[i];
    s = plant_step<STAB, GUST>(e.pv, s, cmd[0], cmd[1], cmd[2], e.tab, nav, e.pv_post, call);
#pragma unroll
    for (int i = 0; i < NX; ++i) e.X[i] = s.v[i];
}

#define DEG2RAD 0.017453292519943295   // numpy deg2rad multiplier (pi/180)
#define RAD2DEG 57.29577951308232      // numpy rad2deg multiplier (180/pi)

__device__ __forceinline__ void apply_fault(int fault, const double* u, double* c)
{
    c[0] = u[0]; c[1] = u[1]; c[2] = u[2];
    if (fault == SERL_FAULT_BE) c[0] = u[0] * 0.3;                                       // envs/be/citation.py:71-75
    else if (fault == SERL_FAULT_JR) c[2] = 15 * 3.14159 / 180;                          // envs/jr/citation.py:71-75
    else if (fault == SERL_FAULT_SA) { const double b = 1.0 * DEG2RAD; c[1] = fmin(fmax(u[1], -b), b); }   // envs/sa :73-79
    else if (fault == SERL_FAULT_SE) { const double b = 2.5 * DEG2RAD; c[0] = fmin(fmax(u[0], -b), b); }   // envs/se :73-79
}

// bind the env's constants (plant variant row, fault shim, reference signals, trim pitch); no dynamics.
// GUST: the kernel instantiation flies the gust schedule (serl_rollout_desc.flags & SERL_ROLLOUT_GUST).  One without it
// carries no trace of the feature, so a gust env bound there is reported (SERL_STATUS_GUST_FLAG) instead of flown as nominal.
// `env` is the row of env_mode / ref_levels / ref_starts: the env index, or actor * n_envs + env in the PER_ACTOR
// instantiations (SERL_ROLLOUT_PER_ACTOR_REFS), whose callers pass that row to env_reset as well.
template <bool GUST>
__device__ __forceinline__ void env_bind(Env& e, const RolloutArgs& a, int env, const real* pv_base, size_t traj)
{
    const int mode = a.env_mode[env];
    const int variant = mode & 0xff;
    e.pv = pv_base + variant * PLANT_NPV;
    const int post = (mode >> 16) & 0xff;
    e.pv_post = post ? pv_base + post * PLANT_NPV : nullptr;
    e.fault = (mode >> 8) & 0xff;
    e.gust = (mode >> 24) & 3;
    e.ref_lv = a.ref_levels + (size_t)env * 2 * SERL_REF_BLOCKS;
    e.ref_st = a.ref_starts + (size_t)env * 2 * SERL_REF_BLOCKS;
    // theta_trim = rad2deg(theta) of reset()'s step output (phlabenv.py:317) — with the sensor-noise shim that output is noisy
    double th0 = plant_ic(variant)[7];
    if (a.sensor_noise) th0 += 4.0 * 1e-3 + 3.2 * 1e-5 * (double)a.sensor_noise[traj * (size_t)(a.horizon + 1) * 7 + 6];
    e.theta_trim = th0 * RAD2DEG;
    if (!GUST && e.gust && a.status) atomicOr(a.status, SERL_STATUS_GUST_FLAG);
}

// observation entries of a kernel instantiation: 7, 10 with incremental control (INC), 2 with symmetric control (SYM).  A
// namespace-scope constant because a local constexpr declaration in a kernel body moved the instruction schedule of the
// instantiations without INC
template <bool INC, bool SYM = false> constexpr int OBS_DIM = SYM ? 2 : INC ? 10 : 7;
// actor outputs: 3, or the elevator alone with symmetric control
template <bool SYM> constexpr int ACT_DIM = SYM ? 1 : 3;
// symmetric control's theta reference offset: the env's constant trim, never replaced by rad2deg(theta0) (phlabenv.py:194, 313)
constexpr double SYM_THETA_TRIM = 0.22;

// a lane without an env: done from the start, with a zero state and observation (it still takes part in the actor)
// INC: incremental control (SERL_ROLLOUT_INCREMENTAL): the observation has 10 entries and the env carries last_u[3], the
// deflection the rates were integrated into (kept by the kernel next to Env, which the other instantiations share unchanged)
// SYM: symmetric control (SERL_ROLLOUT_SYMMETRIC): a 2-entry observation
template <bool INC = false, bool SYM = false>
__device__ __forceinline__ void env_idle(Env& e, const RolloutArgs& a, const real* pv_base, float* obs, double* last_u = nullptr)
{
    e.done = true; e.k = 0; e.ret = 0.0; e.t = 0.0; e.fault = 0; e.gust = 0; e.pv = pv_base; e.pv_post = nullptr; e.theta_trim = 0.0;
    e.ref_lv = a.ref_levels; e.ref_st = a.ref_starts;
#pragma unroll
    for (int i = 0; i < NX; ++i) e.X[i] = 0.0;
#pragma unroll
    for (int i = 0; i < (SYM ? 2 : 7); ++i) obs[i] = 0.f;
    if constexpr (INC)
#pragma unroll
        for (int i = 0; i < 3; ++i) { obs[7 + i] = 0.f; last_u[i] = 0.0; }
}

// end of a trajectory: return and executed steps.  A NaN action poisons the state at once, so a non-finite return or
// state raises SERL_STATUS_NONFINITE.
__device__ __forceinline__ void traj_store(const Env& e, const RolloutArgs& a, size_t traj)
{
    a.returns[traj] = e.ret;
    a.steps[traj] = e.k;
    if (a.status && !isfinite(e.ret + e.X[3] + e.X[7] + e.X[9])) atomicOr(a.status, SERL_STATUS_NONFINITE);
}
__device__ __forceinline__ void track_store(const Env& e, const TrackArgs& tk, size_t traj)
{
#pragma unroll
    for (int c = 0; c < SERL_TRACK_COLS; ++c) tk.out[traj * SERL_TRACK_COLS + c] = e.trk[c];
    if (tk.cost) tk.cost[traj] = (int)e.trk[TRACK_COST];
}

// get_cost (phlabenv.py:369-375, including its degrees-vs-radians comparison on the bank angle) of a step's output x, with
// V0 the airspeed of the plant variant's initial condition
__device__ __forceinline__ bool step_cost(const double* x, double v0)
{
    const double max_phi = 75.0 * DEG2RAD;
    return (fabs(x[4]) * RAD2DEG > 11.0) || (fabs(x[6]) * RAD2DEG > 0.75 * max_phi) || (x[3] < v0 / 3.0);
}

// sensor-noise shim (envs/noise/citation.py:72-82, same model in envs/gust): every native step() output gets
// p,q,r += 3e-5 + 6.3e-4 z; alpha += 4e-10 z; beta += 1.8e-3 + 2.7e-4 z; phi,theta += 4e-3 + 3.2e-5 z  (7 draws per call,
// in that order); the plant's own state is not touched.  call = 0 for reset()'s step, k + 1 for env step k.
__device__ __forceinline__ void sensor_noise(const RolloutArgs& a, size_t traj, int call, double* x)
{
    if (!a.sensor_noise) return;
    const float* z = a.sensor_noise + (traj * (size_t)(a.horizon + 1) + call) * 7;
    x[0] += 3.0 * 1e-5 + 6.3 * 1e-4 * (double)z[0];
    x[1] += 3.0 * 1e-5 + 6.3 * 1e-4 * (double)z[1];
    x[2] += 3.0 * 1e-5 + 6.3 * 1e-4 * (double)z[2];
    x[4] += 4.0 * 1e-10 * (double)z[3];
    x[5] += 1.8 * 1e-3 + 2.7 * 1e-4 * (double)z[4];
    x[6] += 4.0 * 1e-3 + 3.2 * 1e-5 * (double)z[5];
    x[7] += 4.0 * 1e-3 + 3.2 * 1e-5 * (double)z[6];
}

// reset(): initialize(), one zero-command step returns the initial state (phlabenv.py:401-428). obs = [0,0,0,p,q,r,alpha]
// GUST names the same plant_step instance as env_step<STAB, GUST> (call 0 has no gust stage either way), so a kernel
// carries one copy of the step code.
// TRACK: zero the tracking-error sums; the controlled state before step 0 is reset()'s output env.x.
// INC: last_u = 0 and obs[7..9] = last_u (phlabenv.py:425-426)
// SYM: obs = [0, q] (phlabenv.py:422 with obs_idx = [1])
template <bool STAB = false, bool GUST = false, bool TRACK = false, bool INC = false, bool SYM = false>
static __device__ __forceinline__ void env_reset(Env& e, const RolloutArgs& a, int env, float* obs, size_t traj = 0,
                                                 double* last_u = nullptr)
{
    const double* ic = plant_ic(a.env_mode[env] & 0xff);
#pragma unroll
    for (int i = 0; i < NX; ++i) e.X[i] = ic[i];
    double x0[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) x0[i] = e.X[i];
    sensor_noise(a, traj, 0, x0);
    if constexpr (TRACK) {      // env.x before step 0 = reset()'s step output (with the sensor noise of call 0)
#pragma unroll
        for (int c = 0; c < SERL_TRACK_COLS; ++c) e.trk[c] = 0.0;
        e.trk[SERL_TRACK_COLS] = x0[7]; e.trk[SERL_TRACK_COLS + 1] = x0[6]; e.trk[SERL_TRACK_COLS + 2] = x0[5];
        e.trk[TRACK_COST] = 0.0; e.trk[TRACK_V0] = ic[3];
    }
    if constexpr (SYM) {
        obs[0] = 0.f; obs[1] = (float)x0[1];
    } else {
        obs[0] = obs[1] = obs[2] = 0.f;
        obs[3] = (float)x0[0]; obs[4] = (float)x0[1]; obs[5] = (float)x0[2]; obs[6] = (float)x0[4];
    }
    if constexpr (INC)
#pragma unroll
        for (int i = 0; i < 3; ++i) { obs[7 + i] = 0.f; last_u[i] = 0.0; }
    double U[3] = {0.0, 0.0, 0.0}, cmd[3];
    apply_fault(e.fault, U, cmd);
    plant_step_env<STAB, GUST>(e, cmd, a.trace != nullptr, 0);      // call 0: no gust stage
    e.t = 0.0; e.ret = 0.0; e.k = 0; e.done = false;
}

// one CitationEnv.step (phlabenv.py:430-482) + the bookkeeping of Agent.evaluate (agent.py:85-118)
// TRACK: + the tracking error of base/evaluate.py:71-100, e = ref(t) - x_ctrl with x_ctrl = env.x[[7, 6, 5]] when the step
// starts (the native step output of the previous step, or of reset()'s step: in the sensor-noise builds it carries the
// noise, as the reference's env.x does), accumulated in step order in fp64.  With SYM the controlled state is theta alone
// (get_controlled_state of the symmetric env): sum |e_theta|, 0, 0, sum e_theta, e_theta against the trimmed reference
// PER_ACTOR: env_mode holds one row per (actor, env); the replay row's V0 comes from the actor's own replay_env row
// INC: incremental control (phlabenv.py:443-466): the scaled action is a rate (bound 25 deg/s, :205-206), integrated as
// u = last_u + rate * dt in fp64 in the reference's operation order (:377-380; no contraction to fma), u drives the fault
// shim and the plant, last_u = u, obs[7..9] = (float)u; replay rows of SERL_REPLAY_COLS_OF(10) columns
// SYM: symmetric control (phlabenv.py:84-90, 226-231, 304-313, 362-367): `a` holds the elevator alone, the plant takes
// [de, 0, 0] (pad_action), the error is theta's against a reference offset by the constant trim, reward = -|clip(k e_theta)|
// (a sum of one term over error.shape[0] = 1), obs = [e_theta, q]; replay rows of SERL_REPLAY_COLS_SA(2, 1) columns
template <bool STAB = false, bool GUST = false, bool TRACK = false, bool PER_ACTOR = false, bool INC = false, bool SYM = false>
static __device__ __forceinline__ void env_step(Env& e, const RolloutArgs& ar, size_t traj, int actor, bool replay, const float* a, float* obs,
                                                double* last_u = nullptr)
{
    const double bound = INC ? 25.0 * DEG2RAD : 10.0 * DEG2RAD;      // phlabenv.py:205-208
    const double max_theta = 60.0 * DEG2RAD, max_phi = 75.0 * DEG2RAD;
    const double k_err = 6.0 / 3.141592653589793;              // phlabenv.py:226-231
    const double k_err4 = k_err * 4.0;
    double U[3], cmd[3], act_d[3];
    if (ar.action_noise) {
        // action = clip(action + clipped_noise, -1, 1) in float64, then scale_action in float64 (agent.py:90-96)
        const float* nz = ar.action_noise + (traj * ar.horizon + e.k) * ACT_DIM<SYM>;
#pragma unroll
        for (int i = 0; i < ACT_DIM<SYM>; ++i) {
            act_d[i] = fmin(fmax((double)a[i] + (double)nz[i], -1.0), 1.0);
            if constexpr (INC) U[i] = __dadd_rn(-bound, __dmul_rn(0.5 * __dadd_rn(act_d[i], 1.0), bound - (-bound)));
            else U[i] = -bound + 0.5 * (act_d[i] + 1.0) * (bound - (-bound));
        }
    } else {
        // scale_action: low + 0.5*(a + 1.0)*(high - low) with a float32: (a + 1.0) and the halving round in fp32 (:72-73)
#pragma unroll
        for (int i = 0; i < ACT_DIM<SYM>; ++i) {
            act_d[i] = (double)a[i];
            const float t1 = __fadd_rn(a[i], 1.0f);
            const float t2 = __fmul_rn(0.5f, t1);
            if constexpr (INC) U[i] = __dadd_rn(-bound, __dmul_rn((double)t2, bound - (-bound)));
            else U[i] = -bound + (double)t2 * (bound - (-bound));
        }
    }
    if constexpr (INC)
#pragma unroll
        for (int i = 0; i < 3; ++i) U[i] = __dadd_rn(last_u[i], __dmul_rn(U[i], 0.01));
    if constexpr (SYM) { U[1] = U[2] = 0.0; act_d[1] = act_d[2] = 0.0; }      // pad_action (:373-379)
    // a NaN action would be squashed to a bound by the plant's input saturation (as in the reference binary): report it
    if (ar.status && !isfinite(act_d[0] + act_d[1] + act_d[2])) atomicOr(ar.status, SERL_STATUS_NONFINITE);
    apply_fault(e.fault, U, cmd);
    double xo[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) xo[i] = e.X[i];
    plant_step_env<STAB, GUST>(e, cmd, ar.trace != nullptr, (e.k + 1) | (GUST && (e.gust & 1) ? PLANT_CALL_GUST | ((e.gust & 2) ? PLANT_CALL_GUST_UP : 0) : 0));
    sensor_noise(ar, traj, e.k + 1, xo);

    const double t = e.t;
    // + signals.Const(0., t_max, theta_trim) (phlabenv.py:344): the trim offset exists on [0, t_max] only
    const double r_th = ref_deg(e.ref_lv, e.ref_st, t, t <= ar.t_max ? (SYM ? SYM_THETA_TRIM : e.theta_trim) : 0.0, ar.smooth_w) * DEG2RAD;
    const double r_ph = SYM ? 0.0 : ref_deg(e.ref_lv + SERL_REF_BLOCKS, e.ref_st + SERL_REF_BLOCKS, t, 0.0, ar.smooth_w) * DEG2RAD;
    const double e0 = r_th - xo[7], e1 = SYM ? 0.0 : r_ph - xo[6], e2 = SYM ? 0.0 : 0.0 - xo[5];
    if constexpr (TRACK) {
        const double et = r_th - e.trk[SERL_TRACK_COLS], ep = r_ph - e.trk[SERL_TRACK_COLS + 1], eb = 0.0 - e.trk[SERL_TRACK_COLS + 2];
        if constexpr (SYM) {      // a 1-column controlled state: sum |e_theta|, 0, 0, sum e_theta (evaluation.nmae_from_track)
            e.trk[0] += fabs(et); e.trk[3] += et;
        } else {
            e.trk[0] += fabs(et); e.trk[1] += fabs(ep); e.trk[2] += fabs(eb); e.trk[3] += eb;
        }
        e.trk[SERL_TRACK_COLS] = xo[7]; e.trk[SERL_TRACK_COLS + 1] = xo[6]; e.trk[SERL_TRACK_COLS + 2] = xo[5];
        if (step_cost(xo, e.trk[TRACK_V0])) e.trk[TRACK_COST] += 1.0;     // the replay row's cost flag, for every env
    }
    const double c0 = fabs(fmin(fmax(k_err * e0, -1.0), 1.0));
    const double c1 = fabs(fmin(fmax(k_err * e1, -1.0), 1.0));
    const double c2 = fabs(fmin(fmax(k_err4 * e2, -1.0), 1.0));
    double reward = SYM ? -c0 : -((c0 + c1) + c2) / 3.0;
    const bool done = (t >= ar.t_max) || (fabs(xo[7]) > max_theta) || (fabs(xo[6]) > max_phi) || (xo[9] < 50.0);
    if (done) reward += (-1.0 / 0.01) * (ar.t_max - t) * 2.0;  // check_bounds penalty (:391-399)
    e.ret += reward;
    if (ar.actions) {
        float* au = ar.actions + (traj * ar.horizon + e.k) * 3;
        au[0] = (float)U[0]; au[1] = (float)U[1]; au[2] = (float)U[2];
    }
    if (ar.trace) {
        double* tr = ar.trace + (traj * ar.horizon + e.k) * SERL_TRACE_COLS;
#pragma unroll
        for (int i = 0; i < 12; ++i) tr[i] = xo[i];
        tr[12] = U[0]; tr[13] = U[1]; tr[14] = U[2];
        tr[15] = reward;
        tr[16] = act_d[0]; tr[17] = act_d[1]; tr[18] = act_d[2];
        tr[19] = e0; tr[20] = e1; tr[21] = e2;
    }
    const float o0 = (float)e0, o1 = (float)e1, o2 = (float)e2;
    const float o3 = (float)xo[0], o4 = (float)xo[1], o5 = (float)xo[2], o6 = (float)xo[4];
    if (replay) {
        // the transition Agent.evaluate stores (agent.py:101-112) + the cost flag of get_cost (phlabenv.py:369-375,
        // including its degrees-vs-radians comparison on the bank angle).  The same test as step_cost, spelt out: calling
        // it here changes the code of the instantiations without TRACK
        constexpr int S = INC ? 10 : SYM ? 2 : 7;
        float* rp = ar.replay + ((size_t)actor * ar.horizon + e.k) * SERL_REPLAY_COLS_SA(S, ACT_DIM<SYM>);
#pragma unroll
        for (int i = 0; i < S; ++i) rp[i] = obs[i];
        float* rn;
        if constexpr (SYM) {
            rp[S] = (float)act_d[0];
            rn = rp + S + 1;
            rn[0] = o0; rn[1] = o4;
        } else {
            rp[S] = (float)act_d[0]; rp[S + 1] = (float)act_d[1]; rp[S + 2] = (float)act_d[2];
            rn = rp + S + 3;
            rn[0] = o0; rn[1] = o1; rn[2] = o2; rn[3] = o3; rn[4] = o4; rn[5] = o5; rn[6] = o6;
        }
        if constexpr (INC) { rn[7] = (float)U[0]; rn[8] = (float)U[1]; rn[9] = (float)U[2]; }
        rn[S] = (float)reward;
        rn[S + 1] = done ? 1.f : 0.f;
        const int* modes = PER_ACTOR ? ar.env_mode + (size_t)actor * ar.n_envs : ar.env_mode;
        const double v0 = plant_ic(modes[ar.replay_env] & 0xff)[3];
        const bool cost = (fabs(xo[4]) * RAD2DEG > 11.0) || (fabs(xo[6]) * RAD2DEG > 0.75 * max_phi) || (xo[3] < v0 / 3.0);
        rn[S + 2] = cost ? 1.f : 0.f;
    }
    if constexpr (SYM) {
        obs[0] = o0; obs[1] = o4;
    } else {
        obs[0] = o0; obs[1] = o1; obs[2] = o2; obs[3] = o3; obs[4] = o4; obs[5] = o5; obs[6] = o6;
    }
    if constexpr (INC)
#pragma unroll
        for (int i = 0; i < 3; ++i) { last_u[i] = U[i]; obs[7 + i] = (float)U[i]; }
    e.t = t + 0.01;
    e.k += 1;
    e.done = done || (e.k >= ar.horizon);
}

// ---- mbarrier / bulk-copy (TMA) primitives ----------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy executed by the TMA unit; completion is signalled on the mbarrier as transferred bytes
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

