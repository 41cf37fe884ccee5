// K-B0 on tensor cores: CostRegNet's first layer (conv0: 41 -> 8 channels, 3x3x3, 83 of the net's 111 GFLOP at the
// BASELINE config; models.py:757 with ConvBnReLU3D models.py:674-685) as a wgmma GEMM at fp32-grade accuracy.
//
// A 3x3x3 convolution with 8 output channels is a bad implicit GEMM in the usual orientation (M = voxels, N = 8,
// K = 41 * 27): with N = 8 the tensor core idles behind the A-operand traffic.  It is a good one turned inside out:
//
//     Y[p][t * 8 + co] = sum_ci  in[p][ci] * W[co][ci][t]          M = input positions, N = 27 taps x 8 = 216, K = 41
//     out[o][co]       = sum_t   Y[o + off_t][t * 8 + co]            (27 shifted adds per output, done by the epilogue)
//
// so every input position is staged ONCE (K = 41 -> 48 columns of one 128-row operand tile) and multiplied against the
// whole resident weight matrix (224 x 48), and the "im2col" never exists.
//
// fp32-grade accuracy (the volume gate is 1e-4 |v|max): 2-term fp16 operand split, three MMAs per K-step
// (hi*hi + hi*lo + lo*hi into one fp32 accumulator), weights carried x256 (an exact power of two) so that their lo
// terms stay normal fp16 numbers.  The inputs are split unscaled: any |cost| < 65504 stays finite (a x16 scale would
// overflow fp16 at |cost| = 4095).
//
// One persistent CTA per SM walks bricks of 6 x 10 x 24 output voxels (halo brick 8 x 12 x 32 positions = 24 operand
// tiles of 128 positions; a tile = 4 x-rows of 32 positions):
//   warps 4-7  producers : one TMA tensor-map load per tile (box 32 x 4 y 1 z 41 channels = 21 KB fp32, out-of-volume
//                          positions zero-filled by the hardware = the convolution's padding) into a 2-stage ring; then
//                          each thread turns its position's 41 values into the hi / lo fp16 rows of the operand tile
//   warps 0-3  MMA + epilogue warpgroup: per 64-position half of a tile, 9 wgmma (M 64, N 224, K 16) into registers.
//                          A thread then holds all 27 taps of two output channels for two positions and scatters them
//                          into the brick's output tile in shared memory, one tap per step: within a step the
//                          positions map to distinct cells, and a named barrier between steps fixes the accumulation
//                          order => bit-reproducible.  At the end of a brick the tile is written out (raw,
//                          pre-BatchNorm) and the batch statistics accumulated.
// Replaces conv0_k3_kernel (FFMA); same ConvArgs contract (raw output + fixed-point sums).
#include <cuda.h>
#include <cudaTypedefs.h>

#include "conv_common.cuh"
#include "hopper.cuh"

namespace mvsn {

using namespace hop;

namespace c0 {
constexpr int CIN = 41, COUT = 8;
constexpr int BZ = 6, BY = 10, BX = 24;                 // output brick
constexpr int XOFF = 4;                                 // lane of the first output column: the tile's x window starts at x0 - 4,
                                                        // because a TMA box must start 16-byte aligned in the innermost dimension
constexpr int HZ = BZ + 2, HY = BY + 2, HX = 32;        // halo brick (x: one warp = 24 outputs + the two halo columns + 3 + 3 spare)
static_assert(BX % 4 == 0 && XOFF % 4 == 0 && XOFF >= 1 && XOFF + BX + 1 <= HX, "x window");
constexpr int TILES = HZ * HY * HX / 128;               // 24 operand tiles per brick
constexpr int NCOL = 224;                               // 27 taps x 8 channels = 216, padded to a multiple of 16
constexpr float SW = 256.f, INV_SCALE = 1.f / 256.f;
constexpr int W_PART = NCOL * 128;                      // bytes of the hi (or lo) weight image: [224][64] fp16, SW128
constexpr int A_PART = 128 * 128;                       // bytes of the hi (or lo) operand tile
constexpr int OFF_W = 0;                                // hi | lo
constexpr int OFF_A = 2 * W_PART;                       // 2 buffers x (hi | lo)
constexpr int OFF_OUT = OFF_A + 4 * A_PART;             // out_s [8][CSTR] fp32, [BZ][BY][32] per channel
constexpr int CSTR = BZ * BY * 32 + 4;                  // channel stride padded: the four channel pairs of a warp hit distinct banks
constexpr int OUT_FLOATS = COUT * CSTR;
constexpr int STAGE_BYTES = CIN * 128 * 4;              // one TMA box: [41 c][4 y][32 x] fp32 = 20 992 B
constexpr int STAGE_STRIDE = 21504;                     // 128-byte aligned slot
constexpr int OFF_STAGE = OFF_OUT + OUT_FLOATS * 4;     // 2 slots
constexpr int SMEM_BYTES = OFF_STAGE + 2 * STAGE_STRIDE + 1024;
static_assert(OFF_STAGE % 128 == 0 && STAGE_STRIDE % 128 == 0 && STAGE_STRIDE >= STAGE_BYTES, "TMA destinations are 128-byte aligned");
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
constexpr int THREADS = 256;                            // MMA + epilogue warpgroup, 4 producer warps
constexpr int PRODUCER_WARP0 = 4;
static_assert(OFF_A % 1024 == 0 && W_PART % 1024 == 0, "SW128 tiles need 1024-byte alignment");
static_assert(HY % 4 == 0, "a tile is four y-rows of the halo brick");
}  // namespace c0

namespace {

struct SharedC0 {
    uint64_t a_full[2];         // producers (4 warps) -> issuer
    uint64_t a_free[2];         // MMA warpgroup (4 warps) -> producers: the operand tile has been consumed
    uint64_t w_full;
    uint64_t stage_full[2];     // TMA complete_tx -> producers
    uint64_t stage_free[2];     // producers (4 warps) -> TMA thread
};

// one tile of the cost volume: box {32 x, 4 y, 1 z, 41 c} at (x, y, z, 0); coordinates may lie outside the volume (zero fill)
__device__ __forceinline__ void tma_load_tile(void* smem_dst, const CUtensorMap* tmap, int x, int y, int z, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];\n"
        :: "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(x), "r"(y), "r"(z), "r"(0), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void split2_c0(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// MMA + epilogue warpgroup (128 threads).  Accumulator fragment of a 64-row half: d[4 j + 2 hh + e] = Y[row][8 j + 2 q + e]
// with row = 16 w + g + 8 hh (lane = 4 g + q), i.e. column group j = tap, channel co = 2 q + e.
__device__ __forceinline__ void mma_role(const ConvArgs& a, SharedC0& sh, uint8_t* smem, float* out_s, int w, int lane,
                                         int nbricks, int nbx, int nby) {
    using namespace c0;
    const int D = a.Din, H = a.Hin, W = a.Win;
    const int g = lane >> 2, q = lane & 3;
    const uint32_t sbase = smem_u32(smem);
    const uint32_t w_hi = sbase + OFF_W, w_lo = sbase + OFF_W + W_PART;
    float st_s[COUT], st_q[COUT];
#pragma unroll
    for (int c = 0; c < COUT; ++c) st_s[c] = st_q[c] = 0.f;
    mbar_wait(&sh.w_full, 0);
    uint32_t it = 0;
#pragma unroll 1
    for (int b = blockIdx.x; b < nbricks; b += gridDim.x) {
        const int x0 = (b % nbx) * BX, y0 = ((b / nbx) % nby) * BY, z0 = (b / (nbx * nby)) * BZ;
#pragma unroll 1
        for (int m = 0; m < TILES; ++m, ++it) {
            const uint32_t buf = it & 1u;
            mbar_wait(&sh.a_full[buf], (it >> 1) & 1u);
            const int z = m / (HY / 4);
#pragma unroll 1
            for (int h = 0; h < 2; ++h) {
                const uint32_t a_hi = sbase + OFF_A + buf * (2 * A_PART) + h * (A_PART / 2), a_lo = a_hi + A_PART;
                float d[NCOL / 2];
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 3; ++ks) Wgmma<NCOL>::ss(d, desc_sw128(a_hi + ks * 32), desc_sw128(w_lo + ks * 32), ks ? 1 : 0);
#pragma unroll
                for (int ks = 0; ks < 3; ++ks) Wgmma<NCOL>::ss(d, desc_sw128(a_lo + ks * 32), desc_sw128(w_hi + ks * 32), 1);
#pragma unroll
                for (int ks = 0; ks < 3; ++ks) Wgmma<NCOL>::ss(d, desc_sw128(a_hi + ks * 32), desc_sw128(w_hi + ks * 32), 1);
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(d);
                if (h == 1) {                                              // both halves consumed: release the operand tile
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&sh.a_free[buf]);
                }
                // scatter: position (z, y, x) and tap (dy, dz, dx) feed cell (z - dz, y - dy, x + 1 - dx)
                const int r0 = h * 64 + w * 16 + g;                        // rows r0 and r0 + 8: same y row, x and x + 8
                const int y = (m % (HY / 4)) * 4 + (r0 >> 5), x = r0 & 31;
#pragma unroll
                for (int j = 0; j < 27; ++j) {
                    const int dy = j / 9, dz = (j / 3) % 3, dx = j % 3;
                    const int zi = z - dz, yi = y - dy;
                    if ((unsigned)zi < (unsigned)BZ && (unsigned)yi < (unsigned)BY) {
                        float* cell = out_s + (zi * BY + yi) * 32 + 2 * q * CSTR;
#pragma unroll
                        for (int hh = 0; hh < 2; ++hh) {
                            const int xi = x + 8 * hh + 1 - dx;
                            if ((unsigned)xi < 32u) {
                                cell[xi] += d[4 * j + 2 * hh];
                                cell[xi + CSTR] += d[4 * j + 2 * hh + 1];
                            }
                        }
                    }
                    named_bar_sync(1, 128);
                }
            }
        }
        // ---- brick complete: write the raw outputs, accumulate their statistics, clear the tile
        const size_t plane = (size_t)H * W, vol = plane * D;
        const int gx = x0 + lane - XOFF;
        const bool xok = lane >= XOFF && lane < XOFF + BX && gx < W;
#pragma unroll
        for (int co = 0; co < COUT; ++co) {
            float* rows = out_s + co * CSTR + lane;
            float* gout = a.out + (size_t)co * vol + gx;
#pragma unroll 1
            for (int j = w; j < BZ * BY; j += 4) {
                const float v = rows[j * 32] * INV_SCALE;                   // exact: a power of two
                rows[j * 32] = 0.f;
                const int zi = j / BY, yi = j - zi * BY, gz = z0 + zi, gy = y0 + yi;
                if (xok && gz < D && gy < H) {
                    gout[(size_t)gz * plane + (size_t)gy * W] = v;
                    st_s[co] += v; st_q[co] = fmaf(v, v, st_q[co]);
                }
            }
        }
        named_bar_sync(1, 128);                  // every cell cleared before the next brick accumulates
    }
    // batch statistics: fixed order per thread, fixed-order warp reduction, integer (fixed-point) atomics
#pragma unroll
    for (int co = 0; co < COUT; ++co) {
        float s = st_s[co], qq = st_q[co];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, off);
            qq += __shfl_xor_sync(0xffffffffu, qq, off);
        }
        if (lane == 0) {
            unsigned long long* st = reinterpret_cast<unsigned long long*>(a.stats_out) + 2 * co;
            atomicAdd(st, stat_fx(s));
            atomicAdd(st + 1, stat_fx(qq));
        }
    }
}

__global__ void __launch_bounds__(c0::THREADS, 1)
conv0_tc_kernel(const ConvArgs a, const __grid_constant__ CUtensorMap tmap, const uint8_t* __restrict__ wimg) {
    using namespace c0;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ SharedC0 sh;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int D = a.Din, H = a.Hin, W = a.Win;
    const int nbx = (W + BX - 1) / BX, nby = (H + BY - 1) / BY, nbz = (D + BZ - 1) / BZ;
    const int nbricks = nbx * nby * nbz;
    float* out_s = reinterpret_cast<float*>(smem + OFF_OUT);

    if (tid == 0) {
        for (int b = 0; b < 2; ++b) { mbar_init(&sh.a_full[b], 4); mbar_init(&sh.a_free[b], 4); }
        mbar_init(&sh.w_full, 1);
        for (int b = 0; b < 2; ++b) { mbar_init(&sh.stage_full[b], 1); mbar_init(&sh.stage_free[b], 4); }
        fence_barrier_init();
    }
    for (int i = tid; i < OUT_FLOATS; i += THREADS) out_s[i] = 0.f;
    __syncthreads();
    if (tid == 0) {
        mbar_arrive_expect_tx(&sh.w_full, 2u * W_PART);
        bulk_load(smem + OFF_W, wimg, W_PART, &sh.w_full);
        bulk_load(smem + OFF_W + W_PART, wimg + W_PART, W_PART, &sh.w_full);
    }

    auto brick_origin = [&](int b, int& z0, int& y0, int& x0) {
        x0 = (b % nbx) * BX; y0 = ((b / nbx) % nby) * BY; z0 = (b / (nbx * nby)) * BZ;
    };

    if (warp < PRODUCER_WARP0) {
        mma_role(a, sh, smem, out_s, warp, lane, nbricks, nbx, nby);
    } else {
        // =========================== producers: TMA-staged tile -> hi / lo operand rows ====================
        const int row = (warp - PRODUCER_WARP0) * 32 + lane;
        // the first producer warp issues the TMA loads: the whole warp waits for the ring slot (warp-uniform), one elected lane issues
        const bool tma_warp = warp == PRODUCER_WARP0;
        const bool tma_leader = tma_warp ? elect_one() : false;
        auto issue_tma = [&](int b, int m, uint32_t it) {                 // tile (b, m) = the it-th tile of this CTA
            const uint32_t sb = it & 1u;
            mbar_wait(&sh.stage_free[sb], ((it >> 1) & 1u) ^ 1u);
            if (tma_leader) {
                int z0, y0, x0;
                brick_origin(b, z0, y0, x0);
                mbar_arrive_expect_tx(&sh.stage_full[sb], (uint32_t)STAGE_BYTES);
                tma_load_tile(smem + OFF_STAGE + sb * STAGE_STRIDE, &tmap, x0 - XOFF, y0 - 1 + (m % (HY / 4)) * 4, z0 - 1 + m / (HY / 4),
                              &sh.stage_full[sb]);
            }
            __syncwarp();
        };
        uint32_t it = 0;
        int b = blockIdx.x, m = 0;
        if (tma_warp && b < nbricks) issue_tma(b, m, 0);
#pragma unroll 1
        while (b < nbricks) {
            int b2 = b, m2 = m + 1;
            if (m2 == TILES) { m2 = 0; b2 += gridDim.x; }
            if (tma_warp && b2 < nbricks) issue_tma(b2, m2, it + 1);        // the next tile streams in while this one is converted
            const uint32_t sb = it & 1u, buf = it & 1u;
            mbar_wait(&sh.stage_full[sb], (it >> 1) & 1u);
            const float* st = reinterpret_cast<const float*>(smem + OFF_STAGE + sb * STAGE_STRIDE) + row;
            mbar_wait(&sh.a_free[buf], ((it >> 1) & 1u) ^ 1u);
            uint8_t* hi = smem + OFF_A + buf * (2 * A_PART);
#pragma unroll
            for (int k2 = 0; k2 < 3; ++k2) {                               // 16 channels per round: 16 independent loads in flight
                float v[16];
#pragma unroll
                for (int j = 0; j < 16; ++j) v[j] = k2 * 16 + j < CIN ? st[(k2 * 16 + j) * 128] : 0.f;
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    uint32_t h[4], l[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) split2_c0(v[half * 8 + 2 * j], v[half * 8 + 2 * j + 1], h[j], l[j]);
                    const uint32_t off = sw128_offset(row, (k2 * 2 + half) * 8);
                    *reinterpret_cast<uint4*>(hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
                    *reinterpret_cast<uint4*>(hi + A_PART + off) = make_uint4(l[0], l[1], l[2], l[3]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&sh.stage_free[sb]);                 // the staged tile has been consumed
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&sh.a_full[buf]);
            ++it; b = b2; m = m2;
        }
    }
}

// weights [8][41][3][3][3] -> B operand [224 n][64 k = ci] fp16, SWIZZLE_128B, x256, as (hi | lo)
__global__ void pack_conv0_tc_kernel(const float* __restrict__ w, uint8_t* __restrict__ out) {
    using namespace c0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < NCOL * 64; i += gridDim.x * blockDim.x) {
        // column n = ((dy * 3 + dz) * 3 + dx) * 8 + co: the three dz taps of one dy are 72 contiguous accumulator columns
        const int n = i >> 6, k = i & 63, g = n >> 3, co = n & 7;
        const int dy = g / 9, dz = (g / 3) % 3, dx = g % 3, t = dz * 9 + dy * 3 + dx;
        const float v = (n < 27 * COUT && k < CIN) ? w[(size_t)co * CIN * 27 + (size_t)k * 27 + t] * SW : 0.f;
        const __half h = __float2half_rn(v);
        const __half l = __float2half_rn(v - __half2float(h));
        const uint32_t off = sw128_offset(n, k);
        *reinterpret_cast<__half*>(out + off) = h;
        *reinterpret_cast<__half*>(out + W_PART + off) = l;
    }
}

}  // namespace

size_t conv0_tc_workspace_bytes() { return 2 * (size_t)c0::W_PART; }

int launch_conv0_tc(const ConvArgs& a, void* wimg, cudaStream_t st) {
    using namespace c0;
    MVSN_REQUIRE(a.Cin == CIN && a.Cout == COUT, MVSN_EBADSHAPE, "conv0_tc: built for 41 -> 8 channels");
    MVSN_REQUIRE(aligned16(wimg), MVSN_EALIGN, "conv0_tc: weight image must be 16-byte aligned");
    static bool attr_set[64] = {false};
    int dev = 0;
    MVSN_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !attr_set[dev]) {
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(conv0_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        if (dev < 64) attr_set[dev] = true;
    }
    pack_conv0_tc_kernel<<<14, 256, 0, st>>>(a.w, static_cast<uint8_t*>(wimg));
    MVSN_CUDA_CHECK(cudaGetLastError());
    // tensor map of the input [41][D][H][W] fp32 (innermost first); box = one operand tile
    static PFN_cuTensorMapEncodeTiled encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        MVSN_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        MVSN_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, MVSN_ECUDA, "conv0_tc: cuTensorMapEncodeTiled is not available");
        encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(fn);
    }
    MVSN_REQUIRE(a.Win % 4 == 0 && aligned16(a.in0.x), MVSN_EALIGN, "conv0_tc: the input needs 16-byte aligned rows (W %% 4 == 0)");
    CUtensorMap tmap;
    const cuuint64_t gdim[4] = {(cuuint64_t)a.Win, (cuuint64_t)a.Hin, (cuuint64_t)a.Din, (cuuint64_t)CIN};
    const cuuint64_t gstride[3] = {(cuuint64_t)a.Win * 4, (cuuint64_t)a.Win * a.Hin * 4, (cuuint64_t)a.Win * a.Hin * a.Din * 4};
    const cuuint32_t box[4] = {32, 4, 1, (cuuint32_t)CIN}, estr[4] = {1, 1, 1, 1};
    const CUresult cr = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(a.in0.x), gdim, gstride, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    MVSN_REQUIRE(cr == CUDA_SUCCESS, MVSN_ECUDA, "conv0_tc: cuTensorMapEncodeTiled failed (%d)", (int)cr);
    const int nbricks = ((a.Win + BX - 1) / BX) * ((a.Hin + BY - 1) / BY) * ((a.Din + BZ - 1) / BZ);
    const int grid = nbricks < sm_count() ? nbricks : sm_count();
    conv0_tc_kernel<<<grid, THREADS, SMEM_BYTES, st>>>(a, tmap, static_cast<const uint8_t*>(wimg));
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

}  // namespace mvsn
