// tb_probe.cuh -- the probe's four importance-sampling tables on the device (tb200_probe_tables, tb200_set_sky):
// Probe::BuildCDF (src/probe.h:31-79) bit for bit, as snapshot.cpp: build_probe_tables restates it.  Included once,
// by kernels.cu.
//
// BuildCDF's sums are sequential fp32 sums, left to right along each row and then down the row totals; fp32 addition
// is not associative, so neither sum can be a parallel scan.  Rows are independent, so one thread owns one row:
//   k_probe_rows  TB_PROBE_ROWS rows per 32-thread CTA.  The warp stages tiles of TB_PROBE_ROWS x TB_PROBE_TILE texels
//                 in shared memory with cp.async, double-buffered, so that the loads are coalesced and the next tile
//                 is in flight while the row threads sum this one; the row threads write each texel's weight and
//                 running sum into a shared tile the warp stores coalesced into pdfX and cdfX, and each row's total
//                 into pdfY.  A few rows per CTA rather than 32 spread the probe over more SMs: the sum's dependent
//                 chain per tile is the same whatever the number of rows beside it.
//   k_probe_scale one thread per texel: pdfX and cdfX times 1 / the row's total.  Scaling each row in its own CTA
//                 instead left a few hundred warps to stream the tables twice and measured slower than the sums.
//   k_probe_cols  one CTA: thread 0 sums the row totals in order, chunk by chunk through shared memory, into cdfY,
//                 then the CTA divides pdfY and cdfY by the grand total.
// Every operation is an explicit round-to-nearest intrinsic, so that no build flag can contract or reorder it, and
// subnormal texels take part as they are (the build has -ftz=false).  NaN and infinities go through unchanged: a
// black row gives 0 * (1 / 0) = NaN as in the reference.

#define TB_PROBE_ROWS 8
#define TB_PROBE_TILE 128
#define TB_PROBE_CHUNK 4096

// Luminance(Color) * 1, src/maths.h:1571-1574: (r*0.3f + g*0.6f) + b*0.1f
static __device__ __forceinline__ float probe_weight(float4 c)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(c.x, 0.3f), __fmul_rn(c.y, 0.6f)), __fmul_rn(c.z, 0.1f));
}

static __device__ __forceinline__ void probe_cp_async16(void* smem, const void* gmem)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}

// The texels of rows [row0, row0 + rows) and columns [col0, col0 + TB_PROBE_TILE) that exist, into tile[r][c]
static __device__ __forceinline__ void probe_tile_load(const ProbeTablesParams& P, float4 (*tile)[TB_PROBE_TILE + 1], int row0,
                                                       int rows, int col0)
{
    const int cols = min(TB_PROBE_TILE, P.width - col0);
    for (int k = threadIdx.x; k < rows * TB_PROBE_TILE; k += 32) {
        const int r = k / TB_PROBE_TILE, c = k % TB_PROBE_TILE;
        if (c < cols) probe_cp_async16(&tile[r][c], &P.probe[(size_t)(row0 + r) * P.width + col0 + c]);
    }
    asm volatile("cp.async.commit_group;\n" ::: "memory");
}

__global__ void __launch_bounds__(32) k_probe_rows(const __grid_constant__ ProbeTablesParams P)
{
    // +1 element per row: the row threads read and write one column of these tiles at a time, and an unpadded row
    // stride (a multiple of 512 bytes) would put all of them on the same banks
    __shared__ __align__(16) float4 tex[2][TB_PROBE_ROWS][TB_PROBE_TILE + 1];
    __shared__ float wOut[TB_PROBE_ROWS][TB_PROBE_TILE + 1], runOut[TB_PROBE_ROWS][TB_PROBE_TILE + 1];

    const int lane = threadIdx.x;
    const int row0 = blockIdx.x * TB_PROBE_ROWS;
    const int rows = min(TB_PROBE_ROWS, P.height - row0);
    const int tiles = (P.width + TB_PROBE_TILE - 1) / TB_PROBE_TILE;
    float total = 0.0f;   // lane r < rows: the running sum of row row0 + r

    probe_tile_load(P, tex[0], row0, rows, 0);
    for (int t = 0; t < tiles; ++t) {
        const int col0 = t * TB_PROBE_TILE;
        const int cols = min(TB_PROBE_TILE, P.width - col0);
        if (t + 1 < tiles) {
            probe_tile_load(P, tex[(t + 1) & 1], row0, rows, col0 + TB_PROBE_TILE);
            asm volatile("cp.async.wait_group 1;\n" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        }
        __syncthreads();
        if (lane < rows) {
            const float4* texels = tex[t & 1][lane];
            auto step = [&](int c) {
                const float w = probe_weight(texels[c]);
                total = __fadd_rn(total, w);
                wOut[lane][c] = w;
                runOut[lane][c] = total;
            };
            if (cols == TB_PROBE_TILE) {
#pragma unroll 16
                for (int c = 0; c < TB_PROBE_TILE; ++c) step(c);
            } else {
                for (int c = 0; c < cols; ++c) step(c);
            }
        }
        __syncthreads();
        for (int k = lane; k < rows * TB_PROBE_TILE; k += 32) {
            const int r = k / TB_PROBE_TILE, c = k % TB_PROBE_TILE;
            if (c < cols) {
                const size_t i = (size_t)(row0 + r) * P.width + col0 + c;
                P.pdfX[i] = wOut[r][c];
                P.cdfX[i] = runOut[r][c];
            }
        }
        // the next iteration's cp.async overwrites the buffer the row threads have just read, and its row threads
        // the shared outputs the warp has just stored
        __syncthreads();
    }
    if (lane < rows) P.pdfY[row0 + lane] = total;
}

__global__ void __launch_bounds__(256) k_probe_scale(const __grid_constant__ ProbeTablesParams P)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P.width * P.height) return;
    const float inv = __fdiv_rn(1.0f, P.pdfY[i / P.width]);   // the row's 1 / total, as BuildCDF forms it once
    P.pdfX[i] = __fmul_rn(P.pdfX[i], inv);
    P.cdfX[i] = __fmul_rn(P.cdfX[i], inv);
}

__global__ void __launch_bounds__(256) k_probe_cols(const __grid_constant__ ProbeTablesParams P)
{
    __shared__ float run[TB_PROBE_CHUNK];
    __shared__ float grand;
    float total = 0.0f;   // thread 0: the running sum of the row totals
    for (int base = 0; base < P.height; base += TB_PROBE_CHUNK) {
        const int n = min(TB_PROBE_CHUNK, P.height - base);
        for (int i = threadIdx.x; i < n; i += 256) run[i] = P.pdfY[base + i];
        __syncthreads();
        if (threadIdx.x == 0)
            for (int i = 0; i < n; ++i) {
                total = __fadd_rn(total, run[i]);
                run[i] = total;
            }
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += 256) P.cdfY[base + i] = run[i];
        __syncthreads();
    }
    if (threadIdx.x == 0) grand = total;
    __syncthreads();
    for (int i = threadIdx.x; i < P.height; i += 256) {
        P.cdfY[i] = __fdiv_rn(P.cdfY[i], grand);
        P.pdfY[i] = __fdiv_rn(P.pdfY[i], grand);
    }
}

void launch_probe_tables(const ProbeTablesParams& p, cudaStream_t stream, unsigned long long* launchCount)
{
    if (p.width <= 0 || p.height <= 0) return;
    k_probe_rows<<<(unsigned)((p.height + TB_PROBE_ROWS - 1) / TB_PROBE_ROWS), 32, 0, stream>>>(p);
    k_probe_scale<<<(unsigned)(((long long)p.width * p.height + 255) / 256), 256, 0, stream>>>(p);
    k_probe_cols<<<1, 256, 0, stream>>>(p);
    if (launchCount) *launchCount += 3;
}
