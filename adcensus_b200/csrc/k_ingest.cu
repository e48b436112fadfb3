// k_ingest.cu -- stage 1 in cost-input mode (adc_match_cost*): a caller's matching-cost volume becomes the engine's
// [S][H][W][Dp] f32 volume, in one pass over HBM.  Conversion to f32, the transposition of a [D][H][W] volume and the
// value domain of include/adcensus_b200.h (NaN / +inf / >= ADC_COST_MAX -> ADC_COST_MAX, negatives and -0.0 -> +0.0)
// are applied on the way through, so the caller never spends an extra pass on them.  Padding disparities D .. Dp - 1
// get 0.0f, what k_cost_volume writes there.
#include <cuda_fp16.h>

#include "adc_common.cuh"
#include "../../include/adcensus_b200.h"

template <int DT> struct CostIn;
template <> struct CostIn<ADC_COST_F32> {
    using T = float;
    static __device__ __forceinline__ float f32(float v) { return v; }
};
template <> struct CostIn<ADC_COST_F16> {
    using T = unsigned short;
    static __device__ __forceinline__ float f32(unsigned short u) { return __half2float(__ushort_as_half(u)); }
};
template <> struct CostIn<ADC_COST_BF16> {
    using T = unsigned short;
    static __device__ __forceinline__ float f32(unsigned short u) { return __uint_as_float((unsigned)u << 16); }   // exact
};

// The comparisons are written so that NaN fails both: it lands on ADC_COST_MAX, and -0.0 (which is not > 0) on +0.0.
__device__ __forceinline__ float adc_cost_domain(float v) {
    v = v < ADC_COST_MAX ? v : ADC_COST_MAX;
    return v > 0.0f ? v : 0.0f;
}

template <int DT>
__device__ __forceinline__ float ingest_value(const typename CostIn<DT>::T* p) {
    return adc_cost_domain(CostIn<DT>::f32(__ldg(p)));
}

// ---------------------------------------------------------------------------------------------
// [H][W][D]: the source already has d fastest; only the row stride changes (D -> Dp).  A CTA covers IH_PX pixels; the
// threads walk its (pixel, quad) pairs in order, so a warp reads a contiguous run of the source (the four scalar loads of
// a thread hit the same sectors as its neighbours') and writes 512 contiguous bytes with 128-bit stores.
// ---------------------------------------------------------------------------------------------
#define IH_PX 64
#define IH_THREADS 256

template <int DT>
__global__ void __launch_bounds__(IH_THREADS)
k_cost_ingest_hwd(AdcDims dm, const typename CostIn<DT>::T* __restrict__ src, float* __restrict__ vol) {
    const int pair = blockIdx.y, p0 = blockIdx.x * IH_PX;
    const int Q = dm.Dp >> 2;
    const int npx = min(IH_PX, dm.N - p0);
    const typename CostIn<DT>::T* s = src + (size_t)pair * dm.N * dm.D + (size_t)p0 * dm.D;
    float* v = vol + (size_t)pair * dm.vol_stride + (size_t)p0 * dm.Dp;
    for (int i = threadIdx.x; i < npx * Q; i += IH_THREADS) {
        const int px = i / Q, d = 4 * (i - px * Q);
        const typename CostIn<DT>::T* sp = s + (size_t)px * dm.D + d;
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; j++) o[j] = d + j < dm.D ? ingest_value<DT>(sp + j) : 0.0f;
        *reinterpret_cast<float4*>(v + (size_t)px * dm.Dp + d) = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// ---------------------------------------------------------------------------------------------
// [D][H][W]: a transposition.  A CTA stages a tile of ID_PX consecutive pixels x ID_D disparities in shared memory: it is
// loaded row by row (one disparity, ID_PX consecutive pixels: coalesced along x) and written out as one 128-bit store per
// (pixel, quad), eight quads of a pixel from neighbouring lanes.  Row stride ID_PX + 1: a warp's stores into the tile hit
// 32 banks, and the four column reads of a quad (rows 4q .. 4q + 3 of pixel pl, bank (4q + j + pl) mod 32) as well.
// ---------------------------------------------------------------------------------------------
#define ID_PX 64
#define ID_D 32
#define ID_THREADS 256

template <int DT>
__global__ void __launch_bounds__(ID_THREADS)
k_cost_ingest_dhw(AdcDims dm, const typename CostIn<DT>::T* __restrict__ src, float* __restrict__ vol) {
    __shared__ float tile[ID_D][ID_PX + 1];
    const int pair = blockIdx.z, p0 = blockIdx.x * ID_PX, d0 = blockIdx.y * ID_D;
    const typename CostIn<DT>::T* s = src + (size_t)pair * dm.N * dm.D;
    const int lx = threadIdx.x % ID_PX, ly = threadIdx.x / ID_PX;
#pragma unroll
    for (int k = 0; k < ID_D * ID_PX / ID_THREADS; k++) {
        const int dl = ly + k * (ID_THREADS / ID_PX), d = d0 + dl, p = p0 + lx;
        tile[dl][lx] = (d < dm.D && p < dm.N) ? ingest_value<DT>(s + (size_t)d * dm.N + p) : 0.0f;
    }
    __syncthreads();
    float* v = vol + (size_t)pair * dm.vol_stride;
#pragma unroll
    for (int k = 0; k < ID_D * ID_PX / 4 / ID_THREADS; k++) {
        const int i = threadIdx.x + k * ID_THREADS;
        const int q = i % (ID_D / 4), pl = i / (ID_D / 4);
        const int p = p0 + pl, d = d0 + 4 * q;
        if (p < dm.N && d < dm.Dp)
            *reinterpret_cast<float4*>(v + (size_t)p * dm.Dp + d) =
                make_float4(tile[4 * q][pl], tile[4 * q + 1][pl], tile[4 * q + 2][pl], tile[4 * q + 3][pl]);
    }
}

template <int DT>
static void launch_ingest(const AdcDims& dm, int S, int layout, const void* src, float* vol, cudaStream_t st) {
    using T = typename CostIn<DT>::T;
    if (layout == ADC_COST_HWD) {
        dim3 grid((dm.N + IH_PX - 1) / IH_PX, S);
        k_cost_ingest_hwd<DT><<<grid, IH_THREADS, 0, st>>>(dm, static_cast<const T*>(src), vol);
    } else {
        dim3 grid((dm.N + ID_PX - 1) / ID_PX, (dm.Dp + ID_D - 1) / ID_D, S);
        k_cost_ingest_dhw<DT><<<grid, ID_THREADS, 0, st>>>(dm, static_cast<const T*>(src), vol);
    }
}

void adc_launch_cost_ingest(const AdcParams& P, const AdcWave& w, const void* src, int layout, int dtype, float* vol,
                            cudaStream_t st, unsigned long long* launches) {
    switch (dtype) {
        case ADC_COST_F32: launch_ingest<ADC_COST_F32>(P.dm, w.S, layout, src, vol, st); break;
        case ADC_COST_F16: launch_ingest<ADC_COST_F16>(P.dm, w.S, layout, src, vol, st); break;
        default: launch_ingest<ADC_COST_BF16>(P.dm, w.S, layout, src, vol, st); break;
    }
    ++*launches;
}

size_t adc_cost_elem_bytes(int dtype) { return dtype == ADC_COST_F32 ? 4 : 2; }
