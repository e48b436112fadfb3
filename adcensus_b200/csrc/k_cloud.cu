// k_cloud.cu -- point clouds (adc_point_cloud, adc_point_cloud_batch_device).
//
// One pass over n disparity maps that keeps the pixels whose point is finite and inside [z_min, z_max] and writes
// them, in raster order, compacted into each map's output (include/adcensus_b200.h, DESIGN.md section 20): the point
// of cv::reprojectImageTo3D (q_row / coord of k_reproject.cuh, the arithmetic of ADC_REPROJ_POINTS), optionally its
// R, G, B from the map's packed BGR image and its pixel index y*W + x.
//
// Single-pass order-preserving stream compaction with a decoupled look-back:
//   - a CTA takes tiles of CL_TILE consecutive pixels of one map, in the order of a global atomic ticket (ticket t =
//     tile t % tiles of map t / tiles), so every tile it waits for belongs to a CTA that is already running, whatever
//     order the hardware schedules CTAs in; the grid loops over tickets, so any n fits;
//   - each thread reads CL_PER_THREAD disparities (neighbouring lanes, neighbouring pixels), computes their points
//     once in registers and votes its keep bits; one ballot per warp and step and a scan of the 64 counts give every
//     kept pixel its place in the tile;
//   - warp 0 publishes the tile's count (flag AGG), then walks back over the map's earlier tiles 32 at a time, adding
//     counts until it meets a tile whose inclusive prefix is known (flag INCL), and publishes its own inclusive prefix;
//     the map's last tile writes the map's count;
//   - the kept points, colours and pixel indices are staged in shared memory in output order and leave it as
//     consecutive words (colours as bytes), clipped at the map's capacity: every warp store covers one contiguous
//     stretch, and destinations need only 4-byte alignment.
// Workspace: one 64-bit ticket counter and one 64-bit status word per tile of the batch (flag << 32 | count), zeroed by
// a memset before each launch.  Offsets into the batch are 64-bit.
#include <algorithm>

#include "adc_common.cuh"
#include "k_reproject.cuh"

#define CL_THREADS 256
#define CL_PER_THREAD 8
#define CL_TILE (CL_THREADS * CL_PER_THREAD)   // pixels per tile
#define CL_WARPS (CL_THREADS / 32)

static constexpr unsigned long long CL_AGG = 1ull << 32, CL_INCL = 2ull << 32;

static __device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

static __device__ __forceinline__ void st_release(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__global__ void __launch_bounds__(CL_THREADS)
k_point_cloud(int W, int N, int tiles, long long total, const float* __restrict__ disp, const AdcReprojQ Q,
              const uint8_t* __restrict__ bgr, long long bgr_stride, float z_min, float z_max, float* __restrict__ points,
              uint8_t* __restrict__ colors, int* __restrict__ pixels, int* __restrict__ counts, long long cap,
              unsigned long long* __restrict__ work) {
    __shared__ float s_pts[3 * CL_TILE];
    __shared__ int s_pix[CL_TILE];
    __shared__ uint8_t s_rgb[3 * CL_TILE];
    __shared__ int s_off[CL_PER_THREAD * CL_WARPS];   // kept pixels before each (step, warp), in tile order
    __shared__ long long s_ticket;
    __shared__ unsigned s_excl, s_count;
    unsigned long long* const status = work + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned below = (1u << lane) - 1;
    for (;;) {
        if (threadIdx.x == 0) s_ticket = (long long)atomicAdd(work, 1ull);
        __syncthreads();
        const long long t = s_ticket;
        if (t >= total) break;
        const long long m = t / tiles;
        const int tile = (int)(t - m * tiles), r0 = tile * CL_TILE, cnt = min(CL_TILE, N - r0);
        const size_t base = (size_t)m * N + r0;
        float px[CL_PER_THREAD], py[CL_PER_THREAD], pz[CL_PER_THREAD];
        unsigned vote[CL_PER_THREAD];
#pragma unroll
        for (int k = 0; k < CL_PER_THREAD; k++) {
            const int j = k * CL_THREADS + threadIdx.x;
            bool keep = false;
            if (j < cnt) {
                const float d = __ldg(disp + base + j);
                const int r = r0 + j, y = r / W, x = r - y * W;
                const double xd = x, yd = y, dd = d;
                const double ia = __drcp_rn(q_row(Q, 3, xd, yd, dd));
                px[k] = coord(q_row(Q, 0, xd, yd, dd), ia);
                py[k] = coord(q_row(Q, 1, xd, yd, dd), ia);
                pz[k] = coord_z(Q, xd, yd, d, ia);
                keep = isfinite(d) && isfinite(px[k]) && isfinite(py[k]) && isfinite(pz[k]) && z_min <= pz[k] &&
                       pz[k] <= z_max;
            }
            vote[k] = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) s_off[k * CL_WARPS + warp] = __popc(vote[k]);
        }
        __syncthreads();
        if (warp == 0) {
            // exclusive scan of the 64 (step, warp) counts, two per lane, in tile order
            const int a = s_off[2 * lane], b = s_off[2 * lane + 1];
            int incl = a + b;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += v;
            }
            s_off[2 * lane] = incl - a - b;
            s_off[2 * lane + 1] = incl - b;
            const unsigned count = (unsigned)__shfl_sync(0xffffffffu, incl, 31);
            // the map's kept pixels before this tile
            unsigned long long* const st = status + m * tiles;
            unsigned excl = 0;
            if (tile == 0) {
                if (lane == 0) st_release(st, CL_INCL | count);
            } else {
                if (lane == 0) st_release(st + tile, CL_AGG | count);
                for (int pred = tile - 1;; pred -= 32) {
                    const int idx = pred - lane;
                    unsigned long long v = idx >= 0 ? ld_acquire(st + idx) : CL_INCL;
                    while (__any_sync(0xffffffffu, (v >> 32) == 0))
                        if ((v >> 32) == 0) v = ld_acquire(st + idx);
                    const unsigned done = __ballot_sync(0xffffffffu, (v >> 32) == 2);
                    const int stop = done ? __ffs(done) - 1 : 31;   // the nearest tile with an inclusive prefix
                    unsigned sum = lane <= stop ? (unsigned)v : 0u;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                    excl += sum;
                    if (done) break;
                }
                if (lane == 0) st_release(st + tile, CL_INCL | (excl + count));
            }
            if (lane == 0) {
                s_excl = excl;
                s_count = count;
                if (tile == tiles - 1) counts[m] = (int)(excl + count);
            }
        }
        __syncthreads();
        const long long excl = s_excl, count = s_count;
        const uint8_t* const img = colors ? bgr + m * bgr_stride : nullptr;
#pragma unroll
        for (int k = 0; k < CL_PER_THREAD; k++) {
            if (!((vote[k] >> lane) & 1)) continue;
            const int j = k * CL_THREADS + threadIdx.x, q = s_off[k * CL_WARPS + warp] + __popc(vote[k] & below);
            s_pts[3 * q] = px[k];
            s_pts[3 * q + 1] = py[k];
            s_pts[3 * q + 2] = pz[k];
            s_pix[q] = r0 + j;
            if (colors) {
                const uint8_t* c = img + 3 * (size_t)(r0 + j);
                s_rgb[3 * q] = c[2];
                s_rgb[3 * q + 1] = c[1];
                s_rgb[3 * q + 2] = c[0];
            }
        }
        __syncthreads();
        if (excl < cap) {
            const int kept = (int)min(count, cap - excl);
            const size_t o = (size_t)m * cap + excl;
            float* const op = points + 3 * o;
            for (int j = threadIdx.x; j < 3 * kept; j += CL_THREADS) op[j] = s_pts[j];
            if (colors)
                for (int j = threadIdx.x; j < 3 * kept; j += CL_THREADS) colors[3 * o + j] = s_rgb[j];
            if (pixels)
                for (int j = threadIdx.x; j < kept; j += CL_THREADS) pixels[o + j] = s_pix[j];
        }
        __syncthreads();   // the next tile reuses the stage and the ticket
    }
}

static int cloud_tiles(const AdcDims& dm) { return (dm.N + CL_TILE - 1) / CL_TILE; }

size_t adc_point_cloud_work_bytes(const AdcDims& dm, long long n) {
    return n ? 8 * (1 + (size_t)n * (size_t)cloud_tiles(dm)) : 0;
}

void adc_launch_point_cloud(const AdcDims& dm, long long n, const float* disp, const AdcReprojQ& Q, const uint8_t* bgr,
                            long long bgr_stride, float z_min, float z_max, const AdcCloudOut& out, void* work,
                            cudaStream_t st, unsigned long long* launches) {
    const int tiles = cloud_tiles(dm);
    const long long total = n * tiles;
    const unsigned grid = (unsigned)std::min(total, 65535ll);
    k_point_cloud<<<grid, CL_THREADS, 0, st>>>(dm.W, dm.N, tiles, total, disp, Q, bgr, bgr_stride, z_min, z_max,
                                               out.points, out.colors, out.pixels, out.counts, out.capacity,
                                               static_cast<unsigned long long*>(work));
    ++*launches;
}
