// div_exhaustive.cu -- the aggregation's division (adc_recip / adc_div4, adcensus_b200/csrc/adc_div.cuh) on the
// hardware it runs on, against the IEEE quotient.  tests/c/div_sequence.c proves the sequence exact on the CPU for every
// approximate reciprocal within 3 ulp of RN(1/n); only the GPU can say what rcp.approx.ftz.f32 (MUFU.RCP) returns, and
// this program measures that and then runs the real sequence:
//   rcp      for every n in 1..65535: rcp.approx.ftz.f32(n) - __frcp_rn(n) in ulps (minimum, maximum, histogram)
//   binade   for every n in 1..65535 and every mantissa of three binades of x -- [1, 2), the binade of the lower guard
//            1e-30f and the binade of the upper guard 1e30f -- adc_div4 against __fdiv_rn, and __fdiv_rn against the
//            f64 quotient rounded to f32 (53 >= 2 * 24 + 2 bits, so that double rounding is exact: an independent
//            IEEE quotient).  Inside the guarded range every operand and intermediate of the fast path is a normal
//            float or an exact residual, so scaling x by 2^k scales q0, e and q by 2^k exactly and the result is the
//            same for every binade between the guards: [1, 2) stands for all of them.  The two guard binades are
//            where the residual e comes closest to the subnormal range (x near 2^-100, n up to 2^16) and to overflow.
//   guard_x  for all 2^32 patterns of x (in lane u & 3 of the float4, the other lanes 1.0f) and n in {1, 7, 65535,
//            65536}: the fast branch is taken iff x is +0 or in [1e-30f, 1e30f) and n in [1, 65535]
//   guard_n  for all 2^32 patterns of n with x = 1.0f: the fast branch is taken iff n is in [1, 65535]; a NaN n gives
//            NaN in every lane (both branches do, so there the branch cannot be seen and does not matter)
//            Both guard checks see the branch through a reciprocal replaced by NaN: the fast branch turns every lane
//            into NaN, the generic division leaves the 1.0f lanes finite.
//   edge     x at the guards' bit patterns +-1 ulp, every n in 1..65535: the fast sequence (restated below) equals
//            __fdiv_rn, and equals adc_div4 where adc_div4 takes it
//   n_edge   n = 65535 and 65536, every mantissa of the three binades: the fast sequence equals __fdiv_rn
//   sample   4096 (x, n, __fdiv_rn, adc_div4) of the binades, printed for an exact rational check on the CPU
// Every count is printed as "<name> <value>"; the caller asserts on them.  Exit code 0 unless a CUDA call fails.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../adcensus_b200/csrc/adc_div.cuh"

#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) {                                                                      \
            fprintf(stderr, "%s:%d: %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_));     \
            exit(2);                                                                                  \
        }                                                                                             \
    } while (0)

#define NREC 8
#define NHIST 17   // ulp differences -8 .. 8

struct Counts {
    unsigned long long bad;        // adc_div4 (or the fast sequence) != __fdiv_rn
    unsigned long long bad_ref;    // __fdiv_rn != the f64 quotient rounded to f32
    unsigned long long checked;
    unsigned rec[NREC][4];         // first mismatches: x bits, n bits, got bits, want bits
};

__device__ __forceinline__ void record(Counts* c, float x, float n, float got, float want) {
    const unsigned long long i = atomicAdd(&c->bad, 1ull);
    if (i < NREC) {
        c->rec[i][0] = __float_as_uint(x); c->rec[i][1] = __float_as_uint(n);
        c->rec[i][2] = __float_as_uint(got); c->rec[i][3] = __float_as_uint(want);
    }
}

// the body of adc_div4's fast branch for one lane, without the guard
__device__ __forceinline__ float fast_quotient(float x, const AdcRecip& k) {
    const float q0 = __fmaf_rn(k.r, x, 0.0f);
    const float e = __fmaf_rn(-k.n, q0, x);
    return __fmaf_rn(k.r, e, q0);
}

__device__ __forceinline__ float ieee_f64(float x, float n) { return __double2float_rn(__ddiv_rn((double)x, (double)n)); }

// ---- rcp: the hardware reciprocal in ulps of the correctly rounded one -------------------------------------------------
__global__ void k_rcp(int* lo_hi, unsigned long long* hist) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x + 1;
    if (n > 65535) return;
    float r0;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r0) : "f"((float)n));
    const int d = (int)__float_as_uint(r0) - (int)__float_as_uint(__frcp_rn((float)n));
    atomicMin(lo_hi, d);
    atomicMax(lo_hi + 1, d);
    atomicAdd(hist + min(max(d, -8), 8) + 8, 1ull);
}

// ---- binade: every n (blockIdx.y + 1, or the single n given) x every mantissa of the binade at `base` ------------------
#define BN_THREADS 256
#define BN_BLOCKS_X 16
template <bool FAST_ONLY>
__global__ void __launch_bounds__(BN_THREADS) k_binade(unsigned base, float n_fixed, Counts* c) {
    const float n = n_fixed > 0.0f ? n_fixed : (float)(blockIdx.y + 1);
    const AdcRecip k = adc_recip(n);
    unsigned long long bad_ref = 0;
    for (unsigned g = blockIdx.x * BN_THREADS + threadIdx.x; g < (1u << 21); g += BN_BLOCKS_X * BN_THREADS) {
        const float x0 = __uint_as_float(base | 4 * g), x1 = __uint_as_float(base | (4 * g + 1)),
                    x2 = __uint_as_float(base | (4 * g + 2)), x3 = __uint_as_float(base | (4 * g + 3));
        float4 v = make_float4(x0, x1, x2, x3);
        if (FAST_ONLY) v = make_float4(fast_quotient(x0, k), fast_quotient(x1, k), fast_quotient(x2, k), fast_quotient(x3, k));
        else adc_div4(v, k);
        const float x[4] = {x0, x1, x2, x3}, q[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const float want = __fdiv_rn(x[j], n);
            if (__float_as_uint(q[j]) != __float_as_uint(want)) record(c, x[j], n, q[j], want);
            if (!FAST_ONLY) bad_ref += __float_as_uint(want) != __float_as_uint(ieee_f64(x[j], n));
        }
    }
    if (bad_ref) atomicAdd(&c->bad_ref, bad_ref);
    if (threadIdx.x == 0) atomicAdd(&c->checked, (unsigned long long)BN_THREADS * 4 * ((1u << 21) / (BN_BLOCKS_X * BN_THREADS)));
}

// ---- guard: which branch adc_div4 takes -----------------------------------------------------------------------------
__device__ __forceinline__ bool took_fast(float4 v, float n) {
    AdcRecip k = adc_recip(n);
    k.r = __uint_as_float(0x7fc00000u);   // the fast branch now yields NaN in every lane
    adc_div4(v, k);
    return isnan(v.x) && isnan(v.y) && isnan(v.z) && isnan(v.w);
}

__global__ void k_guard_x(float n, Counts* c) {
    const bool n_ok = n >= 1.0f && n <= 65535.0f;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < (1ull << 32);
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned u = (unsigned)i;
        const float x = __uint_as_float(u);
        float4 v = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
        switch (u & 3) { case 0: v.x = x; break; case 1: v.y = x; break; case 2: v.z = x; break; default: v.w = x; }
        const bool want = n_ok && (u == 0u || (u >= 0x0da24260u && u < 0x7149f2cau));   // +0, [1e-30f, 1e30f)
        if (took_fast(v, n) != want) record(c, x, n, want ? 0.0f : 1.0f, want ? 1.0f : 0.0f);
    }
}

__global__ void k_guard_n(Counts* c) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < (1ull << 32);
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const float n = __uint_as_float((unsigned)i);
        if (isnan(n)) {   // both branches give NaN, so the branch cannot be seen (nor does it matter): check the value
            float4 v = make_float4(1.0f, 1.0f, 1.0f, 1.0f);
            adc_div4(v, adc_recip(n));
            if (!(isnan(v.x) && isnan(v.y) && isnan(v.z) && isnan(v.w))) record(c, 1.0f, n, v.x, n);
            continue;
        }
        const bool want = n >= 1.0f && n <= 65535.0f;
        if (took_fast(make_float4(1.0f, 1.0f, 1.0f, 1.0f), n) != want) record(c, 1.0f, n, want ? 0.0f : 1.0f, want ? 1.0f : 0.0f);
    }
}

// ---- edge: the guards' bit patterns +-1 ulp, every n -------------------------------------------------------------------
__global__ void k_edge(Counts* c) {
    const int n_i = blockIdx.x * blockDim.x + threadIdx.x + 1;
    if (n_i > 65535) return;
    const float n = (float)n_i;
    const AdcRecip k = adc_recip(n);
    const unsigned edges[2] = {0x0da24260u, 0x7149f2cau};
    for (int e = 0; e < 2; e++)
        for (int d = -1; d <= 1; d++) {
            const float x = __uint_as_float(edges[e] + d);
            const float f = fast_quotient(x, k), want = __fdiv_rn(x, n);
            if (__float_as_uint(f) != __float_as_uint(want)) record(c, x, n, f, want);
            float4 v = make_float4(x, x, x, x);
            adc_div4(v, k);
            if (__float_as_uint(v.x) != __float_as_uint(want)) record(c, x, n, v.x, want);
            const bool inside = edges[e] + d >= 0x0da24260u && edges[e] + d < 0x7149f2cau;
            if (inside && __float_as_uint(v.x) != __float_as_uint(f)) record(c, x, n, v.x, f);
            atomicAdd(&c->checked, 1ull);
        }
}

// ---- sample: (x, n) pairs for the rational check on the CPU -----------------------------------------------------------
#define NSAMPLE 4096
__global__ void k_sample(const unsigned* bases, unsigned* out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= NSAMPLE) return;
    unsigned long long z = 0x9E3779B97F4A7C15ull * (unsigned long long)(s + 1);
    z = (z ^ (z >> 31)) * 0xBF58476D1CE4E5B9ull;
    z ^= z >> 29;
    const float n = s < 6 ? (s & 1 ? 65536.0f : 65535.0f) : (float)(1 + (unsigned)(z % 65535));
    const float x = __uint_as_float(bases[s % 3] | (unsigned)(z >> 40) & 0x7fffffu);
    float4 v = make_float4(x, x, x, x);
    adc_div4(v, adc_recip(n));
    out[4 * s] = __float_as_uint(x);
    out[4 * s + 1] = __float_as_uint(n);
    out[4 * s + 2] = __float_as_uint(__fdiv_rn(x, n));
    out[4 * s + 3] = __float_as_uint(v.x);
}

// ---- host ----------------------------------------------------------------------------------------------------------------
static Counts* g_c;

static void reset() { CK(cudaMemset(g_c, 0, sizeof(Counts))); }

static void report(const char* name, float ms) {
    CK(cudaDeviceSynchronize());
    Counts h;
    CK(cudaMemcpy(&h, g_c, sizeof(Counts), cudaMemcpyDeviceToHost));
    printf("%s_checked %llu\n%s_bad %llu\n%s_bad_ref %llu\n%s_ms %.1f\n", name, h.checked, name, h.bad, name,
           h.bad_ref, name, ms);
    for (unsigned long long i = 0; i < h.bad && i < NREC; i++)
        printf("%s_first x=%08x n=%08x got=%08x want=%08x\n", name, h.rec[i][0], h.rec[i][1], h.rec[i][2], h.rec[i][3]);
}

template <typename F>
static float timed(F launch) {
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
    CK(cudaEventRecord(a));
    launch();
    CK(cudaGetLastError());
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms = 0.0f;
    CK(cudaEventElapsedTime(&ms, a, b));
    CK(cudaEventDestroy(a));
    CK(cudaEventDestroy(b));
    return ms;
}

int main() {
    const unsigned bases[3] = {0x3f800000u, 0x0d800000u, 0x71000000u};   // [1, 2), 2^-100 .. (1e-30f), 2^99 .. (1e30f)
    const char* names[3] = {"binade_1", "binade_lo", "binade_hi"};
    CK(cudaMalloc(&g_c, sizeof(Counts)));

    int* d_lohi;
    unsigned long long* d_hist;
    CK(cudaMalloc(&d_lohi, 2 * sizeof(int)));
    CK(cudaMalloc(&d_hist, NHIST * sizeof(unsigned long long)));
    const int init[2] = {1 << 30, -(1 << 30)};
    CK(cudaMemcpy(d_lohi, init, sizeof(init), cudaMemcpyHostToDevice));
    CK(cudaMemset(d_hist, 0, NHIST * sizeof(unsigned long long)));
    k_rcp<<<(65535 + 255) / 256, 256>>>(d_lohi, d_hist);
    CK(cudaGetLastError());
    int lohi[2];
    unsigned long long hist[NHIST];
    CK(cudaMemcpy(lohi, d_lohi, sizeof(lohi), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hist, d_hist, sizeof(hist), cudaMemcpyDeviceToHost));
    printf("rcp_ulp_min %d\nrcp_ulp_max %d\n", lohi[0], lohi[1]);
    for (int i = 0; i < NHIST; i++)
        if (hist[i]) printf("rcp_ulp_hist %d %llu\n", i - 8, hist[i]);

    for (int b = 0; b < 3; b++) {
        reset();
        report(names[b], timed([&] { k_binade<false><<<dim3(BN_BLOCKS_X, 65535), BN_THREADS>>>(bases[b], 0.0f, g_c); }));
    }
    reset();
    float ms = timed([&] {
        for (int b = 0; b < 3; b++)
            for (float n : {65535.0f, 65536.0f}) k_binade<true><<<dim3(BN_BLOCKS_X, 1), BN_THREADS>>>(bases[b], n, g_c);
    });
    report("n_edge", ms);
    reset();
    ms = timed([&] { for (float n : {1.0f, 7.0f, 65535.0f, 65536.0f}) k_guard_x<<<4096, 256>>>(n, g_c); });
    report("guard_x", ms);
    reset();
    report("guard_n", timed([&] { k_guard_n<<<4096, 256>>>(g_c); }));
    reset();
    report("edge", timed([&] { k_edge<<<(65535 + 255) / 256, 256>>>(g_c); }));

    unsigned *d_bases, *d_out, out[4 * NSAMPLE];
    CK(cudaMalloc(&d_bases, sizeof(bases)));
    CK(cudaMalloc(&d_out, sizeof(out)));
    CK(cudaMemcpy(d_bases, bases, sizeof(bases), cudaMemcpyHostToDevice));
    k_sample<<<NSAMPLE / 256, 256>>>(d_bases, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, d_out, sizeof(out), cudaMemcpyDeviceToHost));
    for (int s = 0; s < NSAMPLE; s++) printf("sample %08x %08x %08x %08x\n", out[4 * s], out[4 * s + 1], out[4 * s + 2], out[4 * s + 3]);

    CK(cudaFree(d_out));
    CK(cudaFree(d_bases));
    CK(cudaFree(d_hist));
    CK(cudaFree(d_lohi));
    CK(cudaFree(g_c));
    printf("done\n");
    return 0;
}
