// K6 — action-smoothness metric of every trajectory of a rollout (base/core/utils.py:82-120 calc_smoothness), sm_90a.
// Its input is the fp32 action history a rollout writes; it shares no device code with the rollout kernels.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/serl_b200.h"
#include "common.cuh"

// ---- K6: action-smoothness metric (base/core/utils.py:82-120) --------------------------------------------
// One CTA per trajectory: direct DFT of the three actuator signals over the executed steps N (N = 2001 is 3*23*29,
// no radix-2 structure; 12 M fp32 MACs per trajectory), frequency-weighted power summed in double:
//   S = sum_i sum_{k=1}^{N/2-1} f_k |Y_i[k]|^2 dt * 2/N,  f = linspace(dt, 1/(2dt), N/2-1),  result = -sqrt(S)*100*(80/(N dt)).
// The channel means are removed first, as in smoothness_fft_kernel: bin 0 is not part of the metric, and a trimmed
// deflection (a large constant under a small ripple) would otherwise leak through the fp32 twiddles into every bin.
__global__ void __launch_bounds__(256)
smoothness_kernel(const float* __restrict__ actions, const int* __restrict__ steps, int horizon, double dt, double* __restrict__ out)
{
    // one symbol in the three K6 kernels; 128-byte aligned, the work arrays start at 2176 after the static red / mean_s
    // (with 16: at 2064, and smoothness_fft_kernel measured 2 % slower on an H100)
    extern __shared__ __align__(128) unsigned char sm_raw[];
    __shared__ double red[256];
    __shared__ float mean_s[3];
    const int traj = blockIdx.x, tid = threadIdx.x;
    const int N = steps[traj];
    const int M = N / 2 - 1;
    if (M <= 0) { if (tid == 0) out[traj] = -0.0; return; }
    float2* tw = reinterpret_cast<float2*>(sm_raw);            // [N] (cos, sin)(2 pi j / N)
    float* y0 = reinterpret_cast<float*>(tw + horizon);       // [3][N]
    float* y1 = y0 + horizon;
    float* y2 = y1 + horizon;
    const float* a = actions + (size_t)traj * horizon * 3;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int n = tid; n < N; n += 256) { s0 += a[3 * n]; s1 += a[3 * n + 1]; s2 += a[3 * n + 2]; }
    for (int c = 0; c < 3; ++c) {
        red[tid] = c == 0 ? s0 : (c == 1 ? s1 : s2);
        __syncthreads();
        for (int s = 128; s > 0; s >>= 1) { if (tid < s) red[tid] += red[tid + s]; __syncthreads(); }
        if (tid == 0) mean_s[c] = (float)(red[0] / (double)N);
        __syncthreads();
    }
    for (int n = tid; n < N; n += 256) {
        float sv, cv;
        sincospif(2.0f * (float)n / (float)N, &sv, &cv);
        tw[n] = make_float2(cv, sv);
        y0[n] = a[3 * n] - mean_s[0]; y1[n] = a[3 * n + 1] - mean_s[1]; y2[n] = a[3 * n + 2] - mean_s[2];
    }
    __syncthreads();
    const double fstep = M > 1 ? (1.0 / (2.0 * dt) - dt) / (double)(M - 1) : 0.0;
    double acc = 0.0;
    // four frequencies per thread and pass: every y[n] broadcast load feeds 8 fmas per signal
    for (int kb = 1 + 4 * threadIdx.x; kb <= M; kb += 4 * blockDim.x) {
        float re[4][3], im[4][3];
        int idx[4], kk[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            kk[q] = (kb + q <= M) ? kb + q : 0;        // k = 0 is a harmless dummy (weight 0 below)
            idx[q] = 0;
#pragma unroll
            for (int c = 0; c < 3; ++c) { re[q][c] = 0.f; im[q][c] = 0.f; }
        }
        for (int n = 0; n < N; ++n) {
            const float v0 = y0[n], v1 = y1[n], v2 = y2[n];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 w = tw[idx[q]];
                re[q][0] = fmaf(v0, w.x, re[q][0]); im[q][0] = fmaf(v0, w.y, im[q][0]);
                re[q][1] = fmaf(v1, w.x, re[q][1]); im[q][1] = fmaf(v1, w.y, im[q][1]);
                re[q][2] = fmaf(v2, w.x, re[q][2]); im[q][2] = fmaf(v2, w.y, im[q][2]);
                idx[q] += kk[q];
                if (idx[q] >= N) idx[q] -= N;
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (kk[q] == 0) continue;
            double p = 0.0;
#pragma unroll
            for (int c = 0; c < 3; ++c) p += (double)re[q][c] * re[q][c] + (double)im[q][c] * im[q][c];
            acc += (dt + (double)(kk[q] - 1) * fstep) * p;
        }
    }
    red[tid] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (tid < s) red[tid] += red[tid + s];
        __syncthreads();
    }
    if (tid == 0) {
        const double S = red[0] * dt * 2.0 / (double)N;
        out[traj] = -(sqrt(S) * 100.0 * (80.0 / ((double)N * dt)));
    }
}

// ---- K6 (fast path): the same metric through a Bluestein (chirp-z) FFT --------------------------------------------
// N (the episode length) is arbitrary (2001 = 3*23*29 for a full episode, anything for an early termination), so the
// length-N DFT is written as a circular convolution of size FM = 4096 >= 2N-1 with the chirp b[m] = exp(i pi m^2 / N):
//   Y[k] = conj(b[k]) * sum_n (y[n] conj(b[n])) b[k-n]
// = three FFTs of size 4096 = 16^3 in shared memory per transform (three radix-16 passes each; forward DIF: natural -> digit-reversed order; the
// pointwise product with the chirp spectrum in digit-reversed order; inverse DIT: digit-reversed -> natural), O(N log N)
// instead of the O(N^2) of the direct form.  Two real channels share one complex transform (their spectra are separated by
// conjugate symmetry), the channel means are removed first (bin 0 is not part of the metric), phases are reduced exactly
// in integer arithmetic (m^2 mod 2N).  One CTA per trajectory.
#define FM 4096
#define FLOG 12
__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 chirp(int m, int N)      // exp(+i pi m^2 / N)
{
    const int r = (int)(((long long)m * m) % (2 * N));
    float s, c;
    sincospif((float)r / (float)N, &s, &c);
    return make_float2(c, s);
}
// tw[j] = exp(-2 pi i j / FM) for j < FM/2; the upper half of the circle is the negated lower half
__device__ __forceinline__ float2 twiddle(const float2* tw, int j)
{
    const float2 t = tw[j & (FM / 2 - 1)];
    return (j & (FM / 2)) ? make_float2(-t.x, -t.y) : t;
}
// The work arrays are padded by one element per 16 (index i lives at ZI(i)): in the last pass a thread owns 16 CONSECUTIVE
// elements, and without the padding all 32 lanes of a warp would hit the same banks.
#define ZI(i) ((i) + ((i) >> 4))
#define ZN (FM + FM / 16)
__device__ __forceinline__ void dft4(float2 a, float2 b, float2 c, float2 d, float2& x0, float2& x1, float2& x2, float2& x3)
{
    const float2 t0 = make_float2(a.x + c.x, a.y + c.y), t1 = make_float2(a.x - c.x, a.y - c.y);
    const float2 t2 = make_float2(b.x + d.x, b.y + d.y), t3 = make_float2(b.x - d.x, b.y - d.y);
    x0 = make_float2(t0.x + t2.x, t0.y + t2.y); x2 = make_float2(t0.x - t2.x, t0.y - t2.y);     // X1 = t1 - i t3, X3 = t1 + i t3
    x1 = make_float2(t1.x + t3.y, t1.y - t3.x); x3 = make_float2(t1.x - t3.y, t1.y + t3.x);
}
__device__ __forceinline__ void idft4(float2 a, float2 b, float2 c, float2 d, float2& x0, float2& x1, float2& x2, float2& x3)
{
    const float2 t0 = make_float2(a.x + c.x, a.y + c.y), t1 = make_float2(a.x - c.x, a.y - c.y);
    const float2 t2 = make_float2(b.x + d.x, b.y + d.y), t3 = make_float2(b.x - d.x, b.y - d.y);
    x0 = make_float2(t0.x + t2.x, t0.y + t2.y); x2 = make_float2(t0.x - t2.x, t0.y - t2.y);     // x1 = t1 + i t3, x3 = t1 - i t3
    x1 = make_float2(t1.x - t3.y, t1.y + t3.x); x3 = make_float2(t1.x + t3.y, t1.y - t3.x);
}
__device__ __forceinline__ float2 cmulc(float2 a, float2 b) { return cmul(a, make_float2(b.x, -b.y)); }      // a * conj(b)
// forward FFT, decimation in frequency, natural order in, base-4 digit-reversed order out.  FM = 16^3: THREE passes over
// shared memory, each thread (256 of them) transforms 16 elements in registers per pass = two radix-4 stages back to back
// (stage A: span 16q, butterflies over a; stage B: span 4q, butterflies over r; element (a, r) at base + (4a + r) q).
__device__ void fft_dif(float2* z, const float2* tw, int tid)
{
#pragma unroll 1
    for (int lq = FLOG - 4; lq >= 0; lq -= 4) {
        const int q = 1 << lq, tA = FM >> (lq + 4), tB = FM >> (lq + 2);
        const int pos = tid & (q - 1), base = ((tid >> lq) << (lq + 4)) + pos;
        float2 v[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            float2 x0, x1, x2, x3;
            dft4(z[ZI(base + r * q)], z[ZI(base + (4 + r) * q)], z[ZI(base + (8 + r) * q)], z[ZI(base + (12 + r) * q)], x0, x1, x2, x3);
            const int w = (pos + r * q) * tA;
            v[0][r] = x0; v[1][r] = cmul(x1, twiddle(tw, w)); v[2][r] = cmul(x2, twiddle(tw, 2 * w)); v[3][r] = cmul(x3, twiddle(tw, 3 * w));
        }
        const int wb = pos * tB;
        const float2 b1 = twiddle(tw, wb), b2 = twiddle(tw, 2 * wb), b3 = twiddle(tw, 3 * wb);
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            float2 x0, x1, x2, x3;
            dft4(v[a][0], v[a][1], v[a][2], v[a][3], x0, x1, x2, x3);
            z[ZI(base + (4 * a) * q)] = x0;
            z[ZI(base + (4 * a + 1) * q)] = cmul(x1, b1);
            z[ZI(base + (4 * a + 2) * q)] = cmul(x2, b2);
            z[ZI(base + (4 * a + 3) * q)] = cmul(x3, b3);
        }
        __syncthreads();
    }
}
// inverse FFT (unnormalised), decimation in time: digit-reversed order in, natural order out; the mirror image
__device__ void ifft_dit(float2* z, const float2* tw, int tid)
{
#pragma unroll 1
    for (int lq = 0; lq <= FLOG - 4; lq += 4) {
        const int q = 1 << lq, tA = FM >> (lq + 4), tB = FM >> (lq + 2);
        const int pos = tid & (q - 1), base = ((tid >> lq) << (lq + 4)) + pos;
        const int wb = pos * tB;
        const float2 b1 = twiddle(tw, wb), b2 = twiddle(tw, 2 * wb), b3 = twiddle(tw, 3 * wb);
        float2 v[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
            idft4(z[ZI(base + (4 * a) * q)], cmulc(z[ZI(base + (4 * a + 1) * q)], b1), cmulc(z[ZI(base + (4 * a + 2) * q)], b2),
                  cmulc(z[ZI(base + (4 * a + 3) * q)], b3), v[a][0], v[a][1], v[a][2], v[a][3]);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int w = (pos + r * q) * tA;
            float2 x0, x1, x2, x3;
            idft4(v[0][r], cmulc(v[1][r], twiddle(tw, w)), cmulc(v[2][r], twiddle(tw, 2 * w)), cmulc(v[3][r], twiddle(tw, 3 * w)), x0, x1, x2, x3);
            z[ZI(base + r * q)] = x0; z[ZI(base + (4 + r) * q)] = x1; z[ZI(base + (8 + r) * q)] = x2; z[ZI(base + (12 + r) * q)] = x3;
        }
        __syncthreads();
    }
}

// twiddles + the chirp-filter spectrum of a FULL episode (N = horizon), once per launch: most trajectories of a trained
// population run the whole horizon, and for them the filter transform is a fifth of the work
__global__ void __launch_bounds__(256)
smoothness_prep_kernel(int horizon, float2* __restrict__ tw_g, float2* __restrict__ hf_g, float2* __restrict__ cb_g)
{
    extern __shared__ __align__(128) unsigned char sm_raw[];
    float2* hf = reinterpret_cast<float2*>(sm_raw);          // [ZN]
    float2* tw = hf + ZN;                                     // [FM/2]
    const int tid = threadIdx.x;
    for (int j = tid; j < FM / 2; j += 256) {
        float s, c;
        sincospif(-2.0f * (float)j / (float)FM, &s, &c);
        tw[j] = make_float2(c, s);
    }
    for (int m = tid; m < FM; m += 256) {
        const int d = m < horizon ? m : (FM - m < horizon ? FM - m : -1);
        hf[ZI(m)] = d >= 0 ? chirp(d, horizon) : make_float2(0.f, 0.f);
    }
    __syncthreads();
    fft_dif(hf, tw, tid);
    for (int j = tid; j < FM / 2; j += 256) tw_g[j] = tw[j];
    for (int m = tid; m < FM; m += 256) hf_g[m] = hf[ZI(m)];
    for (int m = tid; m <= horizon; m += 256) cb_g[m] = chirp(m, horizon);       // b[m], m = 0 .. N
}

__global__ void __launch_bounds__(256)
smoothness_fft_kernel(const float* __restrict__ actions, const int* __restrict__ steps, int horizon, double dt, double* __restrict__ out,
                      const float2* __restrict__ tw_g, const float2* __restrict__ hf_g, const float2* __restrict__ cb_g)
{
    extern __shared__ __align__(128) unsigned char sm_raw[];
    float2* z = reinterpret_cast<float2*>(sm_raw);            // [ZN] work buffer (padded index ZI)
    float2* hf = z + ZN;                                      // [ZN] spectrum of the chirp filter (digit-reversed order)
    float2* tw = hf + ZN;                                     // [FM/2] twiddles
    __shared__ double red[256];
    __shared__ float mean_s[3];
    const int traj = blockIdx.x, tid = threadIdx.x;
    const int N = steps[traj];
    const int Mb = N / 2 - 1;
    if (Mb <= 0) { if (tid == 0) out[traj] = -0.0; return; }
    const float* a = actions + (size_t)traj * horizon * 3;
    for (int j = tid; j < FM / 2; j += 256) tw[j] = tw_g[j];
    // channel means (bin 0 is excluded from the metric; removing it keeps the float32 transform accurate)
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int n = tid; n < N; n += 256) { s0 += a[3 * n]; s1 += a[3 * n + 1]; s2 += a[3 * n + 2]; }
    for (int c = 0; c < 3; ++c) {
        red[tid] = c == 0 ? s0 : (c == 1 ? s1 : s2);
        __syncthreads();
        for (int s = 128; s > 0; s >>= 1) { if (tid < s) red[tid] += red[tid + s]; __syncthreads(); }
        if (tid == 0) mean_s[c] = (float)(red[0] / (double)N);
        __syncthreads();
    }
    // chirp filter h[m] = b[|m|] for |m| < N (circular), its forward transform stays in hf (full episodes: precomputed)
    if (N == horizon) {
        for (int m = tid; m < FM; m += 256) hf[ZI(m)] = hf_g[m];
        __syncthreads();
    } else {
        for (int m = tid; m < FM; m += 256) {
            const int d = m < N ? m : (FM - m < N ? FM - m : -1);
            hf[ZI(m)] = d >= 0 ? chirp(d, N) : make_float2(0.f, 0.f);
        }
        __syncthreads();
        fft_dif(hf, tw, tid);
    }
    const double fstep = Mb > 1 ? (1.0 / (2.0 * dt) - dt) / (double)(Mb - 1) : 0.0;
    const float inv_m = 1.0f / (float)FM;
    const bool full = N == horizon;              // the chirp b[m] of a full episode comes from the per-launch table
#define K6_CHIRP(m) (full ? cb_g[m] : chirp((m), N))
    double acc = 0.0;
    for (int pass = 0; pass < 2; ++pass) {
        for (int n = tid; n < FM; n += 256) {
            float2 v = make_float2(0.f, 0.f);
            if (n < N) {
                const float re = pass == 0 ? a[3 * n] - mean_s[0] : a[3 * n + 2] - mean_s[2];
                const float im = pass == 0 ? a[3 * n + 1] - mean_s[1] : 0.f;
                const float2 b = K6_CHIRP(n);
                v = cmul(make_float2(re, im), make_float2(b.x, -b.y));
            }
            z[ZI(n)] = v;
        }
        __syncthreads();
        fft_dif(z, tw, tid);
        for (int m = tid; m < FM; m += 256) z[ZI(m)] = cmul(z[ZI(m)], hf[ZI(m)]);
        __syncthreads();
        ifft_dit(z, tw, tid);
        for (int k = 1 + tid; k <= Mb; k += 256) {
            const double f = dt + (double)(k - 1) * fstep;
            if (pass == 0) {
                // T[k] = conj(b[k]) c[k] = Y0[k] + i Y1[k];  Y0 = (T[k] + conj(T[N-k])) / 2,  Y1 = (T[k] - conj(T[N-k])) / (2i)
                const float2 bk = K6_CHIRP(k), bn = K6_CHIRP(N - k);
                float2 tk = cmul(z[ZI(k)], make_float2(bk.x, -bk.y)), tn = cmul(z[ZI(N - k)], make_float2(bn.x, -bn.y));
                tk.x *= inv_m; tk.y *= inv_m; tn.x *= inv_m; tn.y *= inv_m;
                const float y0r = 0.5f * (tk.x + tn.x), y0i = 0.5f * (tk.y - tn.y);
                const float y1r = 0.5f * (tk.y + tn.y), y1i = 0.5f * (tn.x - tk.x);
                acc += f * ((double)y0r * y0r + (double)y0i * y0i + (double)y1r * y1r + (double)y1i * y1i);
            } else {
                const float cr = z[ZI(k)].x * inv_m, ci = z[ZI(k)].y * inv_m;
                acc += f * ((double)cr * cr + (double)ci * ci);
            }
        }
        __syncthreads();
    }
    red[tid] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) { if (tid < s) red[tid] += red[tid + s]; __syncthreads(); }
    if (tid == 0) {
        const double S = red[0] * dt * 2.0 / (double)N;
        out[traj] = -(sqrt(S) * 100.0 * (80.0 / ((double)N * dt)));
    }
}

extern "C" int serl_smoothness(const float* d_actions, const int32_t* d_steps, int32_t n_traj, int32_t horizon, double dt,
                               double* d_out, void* stream)
{
    if (!d_actions || !d_steps || !d_out || n_traj <= 0 || horizon <= 0) return serl_fail(SERL_ERR_ARG, "serl_smoothness: bad argument");
    const cudaStream_t s = (cudaStream_t)stream;
    if (2 * horizon - 1 <= FM) {
        // episodes of up to 2048 steps (training: 2001): Bluestein FFT, O(N log N)
        void* tabs = nullptr;
        const cudaError_t e = serl_scratch(SERL_SCRATCH_K6, s, (size_t)(FM + FM / 2 + FM) * sizeof(float2), &tabs);
        if (e != cudaSuccess) return serl_fail_cuda(e, "smoothness scratch");
        float2* tw_g = (float2*)tabs;
        float2* hf_g = tw_g + FM / 2;
        float2* cb_g = hf_g + FM;
        const int rc = serl_launch("smoothness_prep_kernel", smoothness_prep_kernel, 1, 256, (size_t)(ZN + FM / 2) * sizeof(float2), s,
                                   horizon, tw_g, hf_g, cb_g);
        if (rc != SERL_OK) return rc;
        return serl_launch("smoothness_fft_kernel", smoothness_fft_kernel, n_traj, 256, (size_t)(2 * ZN + FM / 2) * sizeof(float2), s,
                           d_actions, d_steps, horizon, dt, d_out, tw_g, hf_g, cb_g);
    }
    // longer episodes (80 s evaluation mode: 8001 steps): direct DFT
    const size_t smem = (size_t)horizon * (8 + 12);
    if (smem > 200 * 1024) return serl_fail(SERL_ERR_UNSUPPORTED, "serl_smoothness: horizon too long for the shared-memory DFT");
    return serl_launch("smoothness_kernel", smoothness_kernel, n_traj, 256, smem, s, d_actions, d_steps, horizon, dt, d_out);
}
