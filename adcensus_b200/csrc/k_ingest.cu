// k_ingest.cu -- stage 1 in cost-input mode (adc_match_cost*): a caller's matching-cost volume becomes the engine's
// [S][H][W][Dp] f32 volume, in one pass over HBM.  Conversion to f32, the transposition of a [D][H][W] volume and the
// value domain of include/adcensus_b200.h (NaN / +inf / >= ADC_COST_MAX -> ADC_COST_MAX, negatives and -0.0 -> +0.0)
// are applied on the way through, so the caller never spends an extra pass on them.  Padding disparities D .. Dp - 1
// get 0.0f, what k_cost_volume writes there.  The second half of the file is the way back out: the export kernels
// (adc_match_volumes*) write one of the engine's volumes to a caller's buffer in the same layouts and element types.
#include <cuda_bf16.h>
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

// =============================================================================================
// Volume export (adc_match_volumes*): the mirror of ingestion.  One pass from the engine's [S][H][W][Dp] f32 volume to the
// caller's buffer, pair i of the wave at element i*H*W*D, in [H][W][D] or [D][H][W], as f32 (a bit copy), f16 or bf16.
// Rounding: f16 is IEEE round-to-nearest-even (__float2half_rn: values >= 65520 become +inf), as torch's .half() and
// numpy's astype(float16); bf16 is round-to-nearest-even (__float2bfloat16_rn).  The engine's volumes hold no NaN (every
// cost is finite and >= +0: the AD-census cost by construction, a caller's cost after the value domain, and
// aggregation / scanline optimisation only sum, halve and divide those), so no NaN rule is needed.
// Destinations need only be aligned to their element size: where a vector store would straddle an alignment boundary
// the kernels fall back to narrower stores, decided from the address itself.  Element offsets are 64-bit (one
// 1920x1080x192 volume is 398 M elements).
// ---------------------------------------------------------------------------------------------
template <int DT> struct CostOut;
template <> struct CostOut<ADC_COST_F32> {
    using T = float;
    static __device__ __forceinline__ float cvt(float v) { return v; }
};
template <> struct CostOut<ADC_COST_F16> {
    using T = unsigned short;
    static __device__ __forceinline__ unsigned short cvt(float v) { return __half_as_ushort(__float2half_rn(v)); }
};
template <> struct CostOut<ADC_COST_BF16> {
    using T = unsigned short;
    static __device__ __forceinline__ unsigned short cvt(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
};

// ---------------------------------------------------------------------------------------------
// [H][W][D]: strips the Dp padding.  A CTA covers px pixels (a multiple of 4, about 4096 elements), i.e. a contiguous
// run of px*D destination elements; since p0*D is a multiple of 4, every CTA of a pair starts at the same phase relative
// to a 4-element boundary.  The threads walk the run in groups of 4 elements starting at the first 4-element-aligned
// address (16-byte stores for f32, 8-byte stores of four packed values for f16 / bf16); the at most 3 elements before
// that address and 3 after the last whole group go out as scalars.  The loads are the 4 consecutive source floats of a
// group (crossing a pixel boundary where the group does): neighbouring lanes read neighbouring runs of the source.
// ---------------------------------------------------------------------------------------------
#define EH_THREADS 256
#define EH_ELEMS 4096

template <int DT>
__global__ void __launch_bounds__(EH_THREADS)
k_cost_export_hwd(AdcDims dm, int px, const float* __restrict__ vol, typename CostOut<DT>::T* __restrict__ dst) {
    using T = typename CostOut<DT>::T;
    constexpr unsigned ALIGN = 4 * sizeof(T);
    const int pair = blockIdx.y, p0 = blockIdx.x * px;
    const unsigned D = (unsigned)dm.D;
    const int L = min(px, dm.N - p0) * dm.D;
    const float* v = vol + (size_t)pair * dm.vol_stride + (size_t)p0 * dm.Dp;
    T* o = dst + ((size_t)pair * dm.N + p0) * dm.D;
    const int head = min(L, (int)(((ALIGN - ((unsigned)(uintptr_t)o & (ALIGN - 1))) & (ALIGN - 1)) / sizeof(T)));
    const int G = (L - head) / 4, tail0 = head + 4 * G;
    for (int g = threadIdx.x; g < G; g += EH_THREADS) {
        const unsigned l = head + 4 * g;
        unsigned p = l / D, d = l - p * D;
        T x[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            x[j] = CostOut<DT>::cvt(v[(size_t)p * dm.Dp + d]);
            if (++d == D) { d = 0; ++p; }
        }
        if constexpr (DT == ADC_COST_F32)
            *reinterpret_cast<float4*>(o + l) = make_float4(x[0], x[1], x[2], x[3]);
        else
            *reinterpret_cast<uint2*>(o + l) = make_uint2(x[0] | (unsigned)x[1] << 16, x[2] | (unsigned)x[3] << 16);
    }
    // threads 0..head-1: the head, threads 32..: the tail (each fewer than 4 elements)
    const int t = threadIdx.x;
    const int l = t < head ? t : (t >= 32 && tail0 + t - 32 < L ? tail0 + t - 32 : -1);
    if (l >= 0) {
        const unsigned p = (unsigned)l / D, d = (unsigned)l - p * D;
        o[l] = CostOut<DT>::cvt(v[(size_t)p * dm.Dp + d]);
    }
}

// ---------------------------------------------------------------------------------------------
// [D][H][W]: a transposition, the inverse of k_cost_ingest_dhw.  A CTA stages ED_PX consecutive pixels x ED_D
// disparities: loaded with one 128-bit load per (pixel, quad), the eight quads of a pixel from neighbouring lanes (a warp
// reads four whole 128-byte pixel runs), and written out one disparity row per warp store, coalesced along x.
// The tile has row stride ED_PX = 128 floats and no padding; pixel pl of row r sits in column pl ^ (4 * (r >> 2)), an XOR
// swizzle by the row's quad that keeps neighbouring pixels pairwise together (the XOR mask is a multiple of 4 below 32).
//  * Tile stores: a warp's lanes are quads q = lane % 8 of pixels pl = pl0 + lane / 8 (pl0 a multiple of 4), and for
//    component j all of them write row 4q + j: bank = (pl ^ 4q) mod 32 = ((pl0 mod 32) ^ 4q) + lane / 8, where the first
//    term runs over the 8 multiples of 4 and the second over 0..3: 32 distinct banks.
//  * Row reads: a row is two 64-pixel segments; in each, lane reads pixels 2*lane, 2*lane + 1 as one 64-bit float2 (the
//    swizzle keeps the pair adjacent and 8-byte aligned, and XOR with a mask below 32 permutes each 32-word block), so
//    each half-warp reads a permutation of 32 consecutive words: conflict-free.
// Stores: one word of two pixels per lane, 8 bytes for f32 and 4 bytes for f16 / bf16, a warp covering a 64-pixel
// segment.  When a segment's destination starts one element past a word boundary (H*W odd, or a base offset), the words
// hold pixels (2k - 1, 2k): lane k takes pixel 2k - 1 from lane k - 1 by a shuffle, and the first and last pixel of the
// segment go out as single-element stores.
// ---------------------------------------------------------------------------------------------
#define ED_PX 128
#define ED_D 32
#define ED_THREADS 256

template <int DT>
__device__ __forceinline__ void store_pair(typename CostOut<DT>::T* o, typename CostOut<DT>::T a, typename CostOut<DT>::T b) {
    if constexpr (DT == ADC_COST_F32) *reinterpret_cast<float2*>(o) = make_float2(a, b);
    else *reinterpret_cast<unsigned*>(o) = a | (unsigned)b << 16;
}

template <int DT>
__global__ void __launch_bounds__(ED_THREADS)
k_cost_export_dhw(AdcDims dm, const float* __restrict__ vol, typename CostOut<DT>::T* __restrict__ dst) {
    using T = typename CostOut<DT>::T;
    __shared__ __align__(16) float tile[ED_D][ED_PX];
    const int pair = blockIdx.z, p0 = blockIdx.x * ED_PX, d0 = blockIdx.y * ED_D;
    const float* v = vol + (size_t)pair * dm.vol_stride;
#pragma unroll
    for (int k = 0; k < ED_D * ED_PX / 4 / ED_THREADS; k++) {
        const int i = threadIdx.x + k * ED_THREADS;
        const int q = i % (ED_D / 4), pl = i / (ED_D / 4);
        const int p = p0 + pl, d = d0 + 4 * q;
        float4 x = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (p < dm.N && d < dm.Dp) x = *reinterpret_cast<const float4*>(v + (size_t)p * dm.Dp + d);
        const int c = pl ^ (4 * q);
        tile[4 * q][c] = x.x;
        tile[4 * q + 1][c] = x.y;
        tile[4 * q + 2][c] = x.z;
        tile[4 * q + 3][c] = x.w;
    }
    __syncthreads();
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    for (int r = warp; r < ED_D && d0 + r < dm.D; r += ED_THREADS / 32) {
        const int sw = 4 * (r >> 2);
#pragma unroll
        for (int sg = 0; sg < ED_PX / 64; sg++) {
            const int npx = min(64, dm.N - p0 - 64 * sg);      // pixels of this segment (uniform over the warp)
            if (npx <= 0) break;
            T* o = dst + ((size_t)pair * dm.D + d0 + r) * dm.N + p0 + 64 * sg;
            const float2 f = *reinterpret_cast<const float2*>(&tile[r][(64 * sg + 2 * lane) ^ sw]);
            const T lo = CostOut<DT>::cvt(f.x), hi = CostOut<DT>::cvt(f.y);   // pixels 2*lane, 2*lane + 1
            if (((uintptr_t)o & sizeof(T)) == 0) {
                if (2 * lane + 1 < npx) store_pair<DT>(o + 2 * lane, lo, hi);
                else if (2 * lane < npx) o[2 * lane] = lo;
            } else {
                const T prev = __shfl_up_sync(0xffffffffu, hi, 1);              // pixel 2*lane - 1
                if (lane == 0) o[0] = lo;
                else if (2 * lane < npx) store_pair<DT>(o + 2 * lane - 1, prev, lo);
                else if (2 * lane - 1 < npx) o[2 * lane - 1] = prev;
                if (lane == 31 && npx == 64) o[63] = hi;
            }
        }
    }
}

static int export_px(const AdcDims& dm) { return ((EH_ELEMS + dm.D - 1) / dm.D + 3) & ~3; }

template <int DT>
static void launch_export(const AdcDims& dm, int S, int layout, const float* vol, void* dst, cudaStream_t st) {
    using T = typename CostOut<DT>::T;
    if (layout == ADC_COST_HWD) {
        const int px = export_px(dm);
        dim3 grid((dm.N + px - 1) / px, S);
        k_cost_export_hwd<DT><<<grid, EH_THREADS, 0, st>>>(dm, px, vol, static_cast<T*>(dst));
    } else {
        dim3 grid((dm.N + ED_PX - 1) / ED_PX, (dm.D + ED_D - 1) / ED_D, S);
        k_cost_export_dhw<DT><<<grid, ED_THREADS, 0, st>>>(dm, vol, static_cast<T*>(dst));
    }
}

void adc_launch_cost_export(const AdcParams& P, const AdcWave& w, const float* vol, void* dst, int layout, int dtype,
                            cudaStream_t st, unsigned long long* launches) {
    switch (dtype) {
        case ADC_COST_F32: launch_export<ADC_COST_F32>(P.dm, w.S, layout, vol, dst, st); break;
        case ADC_COST_F16: launch_export<ADC_COST_F16>(P.dm, w.S, layout, vol, dst, st); break;
        default: launch_export<ADC_COST_BF16>(P.dm, w.S, layout, vol, dst, st); break;
    }
    ++*launches;
}
