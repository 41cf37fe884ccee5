// Importance sampling from a density grid (mvsn_sample_importance): ray_marcher_fine and sample_pdf
// (data/ray_utils.py:98-141, :199-224) for a batch of rays, one warp per ray.
//
// Per ray, with S coarse depths z_j (marched, or the caller's) and their NDC:
//   sigma_j   trilinear lookup of the grid at the sample's NDC (align_corners, zero padding), the render's own
//             trilinear_corners arithmetic
//   alpha_j = 1 - exp(-relu(sigma_j)) (as -expm1: no cancellation for small sigma), T_j = prod_{i<j} (1 - alpha_i +
//             1e-10), w_j = alpha_j T_j
//   cdf       [0, cumsum((w_1..w_{S-2} + 1e-5) / sum)]        (S - 1 values)
//   bins      (z_j + z_{j+1}) / 2                              (S - 1 values)
//   K fine    searchsorted(cdf, u, right) -> below / above -> bins[below] + t (bins[above] - bins[below])
//   output    sort(cat(fine, coarse)), pts = o + d z (unfused, as torch rounds it), optionally the NDC.
// Lane l owns the contiguous coarse samples [l s, (l + 1) s), s = ceil(S / 32), for the two scans (a multiplicative
// one for T, an additive one for the cdf: sequential inside a lane, shuffles across lanes); the per-sample passes are
// strided.  The S + K outputs are sorted by a bitonic network over the next power of two in shared memory, on keys whose
// unsigned order is the float order with every NaN last, as torch.sort orders them; the coarse values pass through
// bit-exactly.
#include "render_frontend.cuh"

namespace mvsn {

namespace imp {
constexpr int WARPS = 4;                                 // rays per CTA
constexpr unsigned FULL = 0xffffffffu;
static int pow2_at_least(int n) { int p = 1; while (p < n) p <<= 1; return p; }
static int s_pad(int S) { return (S + 3) & ~3; }
// per warp: A [s_pad(S)] (alpha, then bins) | B [s_pad(S)] (weights, then cdf) | keys [pow2(S + K)] (coarse z, then keys)
static size_t smem_bytes(int S, int K) { return (size_t)WARPS * (2 * s_pad(S) + pow2_at_least(S + K)) * sizeof(float); }
}  // namespace imp

__device__ __forceinline__ uint32_t sort_key(float f) {
    const uint32_t b = __float_as_uint(f);
    if (f != f) return 0xffffffffu;                      // NaN: after +inf (and equal to the padding)
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
    if (k == 0xffffffffu) return __uint_as_float(0x7fffffffu);
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// torch.linspace(0, 1, K)[k]: step = 1 / (K - 1), the first half counted up from 0, the second down from 1
__device__ __forceinline__ float linspace_u(int k, int K) {
    if (K == 1) return 0.f;
    const float step = __fdiv_rn(1.f, (float)(K - 1));
    return k < K / 2 ? __fmul_rn(step, (float)k) : __fsub_rn(1.f, __fmul_rn(step, (float)(K - 1 - k)));
}

// F.grid_sample of the [D][Hp][Wp] grid at an NDC point (align_corners=True, zero padding), corners x fastest
__device__ __forceinline__ float grid_sigma(const SceneDev& g, const float* __restrict__ sigma, float nx, float ny,
                                            float nz) {
    const Trilinear t = trilinear_corners(g, nx, ny, nz);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int x = t.x0 + (c & 1), y = t.y0 + ((c >> 1) & 1), z = t.z0 + (c >> 2);
        if ((unsigned)x < (unsigned)g.Wp && (unsigned)y < (unsigned)g.Hp && (unsigned)z < (unsigned)g.D)
            s = fmaf(__ldg(sigma + ((size_t)z * g.Hp + y) * g.Wp + x), t.wx[c & 1] * t.wy[(c >> 1) & 1] * t.wz[c >> 2], s);
    }
    return s;
}

__device__ __forceinline__ float warp_exclusive_product(float p, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float q = __shfl_up_sync(imp::FULL, p, o);
        if (lane >= o) p *= q;
    }
    const float e = __shfl_up_sync(imp::FULL, p, 1);
    return lane == 0 ? 1.f : e;
}
__device__ __forceinline__ float warp_exclusive_sum(float s, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float q = __shfl_up_sync(imp::FULL, s, o);
        if (lane >= o) s += q;
    }
    const float e = __shfl_up_sync(imp::FULL, s, 1);
    return lane == 0 ? 0.f : e;
}

// MARCH: the coarse samples are ray_z / ray_z_jittered of the ray's near / far (the fine-tuning backward's march) and
// their NDC ndc_of_point<true>; otherwise io.z_in / io.ndc_in.
template <bool MARCH>
__global__ void __launch_bounds__(imp::WARPS * 32) importance_kernel(const SceneDev sc, const RayGenDev rg,
                                                                     const ImportanceIO io) {
    extern __shared__ __align__(16) float smem[];
    __shared__ Cams cams;
    if (io.cams) load_cams(sc, &cams, threadIdx.x);
    __syncthreads();
    const int S = io.S, K = io.K, M = S + K;
    int P = 4;
    while (P < M) P <<= 1;
    const int SP = (S + 3) & ~3;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* A = smem + (size_t)warp * (2 * SP + P);
    float* B = A + SP;
    uint32_t* keys = reinterpret_cast<uint32_t*>(B + SP);
    float* zc = reinterpret_cast<float*>(keys);
    const int seg = (S + 31) / 32, b0 = min(S, lane * seg), b1 = min(S, b0 + seg);
    for (int ray = blockIdx.x * imp::WARPS + warp; ray < io.N; ray += gridDim.x * imp::WARPS) {
        const float4* rp = reinterpret_cast<const float4*>(io.rays + (size_t)ray * 8);
        const float4 r0 = __ldg(rp), r1 = __ldg(rp + 1);
        // ---- coarse samples and their alpha ----
        for (int j = lane; j < S; j += 32) {
            const size_t si = (size_t)ray * S + j;
            float z, nx, ny, nz;
            if (MARCH) {
                z = io.jitter ? ray_z_jittered(r1.z, r1.w, io.t_steps, j, S, rg.lindisp, __ldg(io.jitter + si))
                              : ray_z(r1.z, r1.w, __ldg(io.t_steps + j), rg.lindisp);
                const float px = __fadd_rn(r0.x, __fmul_rn(r0.w, z)), py = __fadd_rn(r0.y, __fmul_rn(r1.x, z)),
                            pz = __fadd_rn(r0.z, __fmul_rn(r1.y, z));
                ndc_of_point<true>(sc, cams, rg, px, py, pz, nx, ny, nz);
            } else {
                z = __ldg(io.z_in + si);
                nx = __ldg(io.ndc_in + 3 * si); ny = __ldg(io.ndc_in + 3 * si + 1); nz = __ldg(io.ndc_in + 3 * si + 2);
            }
            zc[j] = z;
            A[j] = -expm1f(-fmaxf(grid_sigma(sc, io.sigma, nx, ny, nz), 0.f));   // 1 - exp(-relu(sigma)), no cancellation
        }
        __syncwarp();
        // ---- transmittance, weights + 1e-5 (w_1 .. w_{S-2}; 0 elsewhere) and their sum ----
        float p = 1.f;
        for (int j = b0; j < b1; ++j) p *= (1.f - A[j]) + 1e-10f;
        float T = warp_exclusive_product(p, lane), vs = 0.f;
        for (int j = b0; j < b1; ++j) {
            const float a = A[j];
            const float v = (j >= 1 && j <= S - 2) ? __fadd_rn(__fmul_rn(a, T), 1e-5f) : 0.f;
            B[j] = v;
            vs += v;
            T *= (1.f - a) + 1e-10f;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) vs += __shfl_xor_sync(imp::FULL, vs, o);
        // ---- cdf[i] = sum_{j <= i} v_j / sum, i = 0 .. S - 2 (cdf[0] = 0) ----
        float cs = 0.f;
        for (int j = b0; j < b1; ++j) cs += __fdiv_rn(B[j], vs);
        float c = warp_exclusive_sum(cs, lane);
        for (int j = b0; j < b1; ++j) {
            c += __fdiv_rn(B[j], vs);
            B[j] = c;
        }
        __syncwarp();
        // ---- bins (over alpha, consumed) ----
        for (int i = lane; i < S - 1; i += 32) A[i] = __fmul_rn(0.5f, __fadd_rn(zc[i], zc[i + 1]));
        __syncwarp();
        // ---- keys: the coarse depths in place, the K fine samples behind them, the padding ----
        for (int j = lane; j < S; j += 32) keys[j] = sort_key(zc[j]);
        for (int k = lane; k < K; k += 32) {
            const float u = io.u ? __ldg(io.u + (size_t)ray * K + k) : linspace_u(k, K);
            int lo = 0, hi = S - 1;                             // searchsorted(cdf, u, right=True)
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (B[mid] <= u) lo = mid + 1; else hi = mid;
            }
            const int below = max(0, lo - 1), above = min(S - 2, lo);
            const float cb = B[below];
            float den = __fsub_rn(B[above], cb);
            if (den < 1e-5f) den = 1.f;
            const float t = __fdiv_rn(__fsub_rn(u, cb), den);
            const float lo_bin = A[below];
            keys[S + k] = sort_key(__fadd_rn(lo_bin, __fmul_rn(t, __fsub_rn(A[above], lo_bin))));
        }
        for (int m = M + lane; m < P; m += 32) keys[m] = 0xffffffffu;
        __syncwarp();
        // ---- bitonic sort, ascending ----
        for (int k = 2; k <= P; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int t = lane; t < P / 2; t += 32) {
                    const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), l = i + j;
                    const uint32_t a = keys[i], b = keys[l];
                    if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[l] = a; }
                }
                __syncwarp();
            }
        }
        // ---- outputs ----
        for (int m = lane; m < M; m += 32) {
            const float z = key_value(keys[m]);
            const size_t o = (size_t)ray * M + m;
            io.z_out[o] = z;
            const float px = __fadd_rn(r0.x, __fmul_rn(r0.w, z)), py = __fadd_rn(r0.y, __fmul_rn(r1.x, z)),
                        pz = __fadd_rn(r0.z, __fmul_rn(r1.y, z));
            io.pts_out[3 * o] = px; io.pts_out[3 * o + 1] = py; io.pts_out[3 * o + 2] = pz;
            if (io.ndc_out) {
                float nx, ny, nz;
                ndc_of_point<true>(sc, cams, rg, px, py, pz, nx, ny, nz);
                io.ndc_out[3 * o] = nx; io.ndc_out[3 * o + 1] = ny; io.ndc_out[3 * o + 2] = nz;
            }
        }
        __syncwarp();
    }
}

int launch_importance(const SceneDev& sc, const RayGenDev& rg, const ImportanceIO& io, cudaStream_t stream) {
    const size_t smem = imp::smem_bytes(io.S, io.K);
    static bool attr_set[64] = {false};                   // once per device, not per launch
    int dev = 0;
    MVSN_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !attr_set[dev]) {
        const int max_smem = (int)imp::smem_bytes(MAX_IMPORTANCE_SAMPLES - 1, 1);
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(importance_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(importance_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
        if (dev < 64) attr_set[dev] = true;
    }
    const int ctas = cdiv(io.N, imp::WARPS), cap = 16 * sm_count();
    const int grid = ctas < cap ? ctas : cap;
    if (grid <= 0) return MVSN_OK;
    if (io.t_steps) importance_kernel<true><<<grid, imp::WARPS * 32, smem, stream>>>(sc, rg, io);
    else            importance_kernel<false><<<grid, imp::WARPS * 32, smem, stream>>>(sc, rg, io);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

}  // namespace mvsn
