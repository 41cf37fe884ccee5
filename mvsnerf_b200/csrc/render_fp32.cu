// K-C, fp32 mode: the fused per-ray render kernel with the MLP on the fp32 FFMA pipe.
//
// One persistent CTA per SM; a CTA walks over tiles of 128 samples (one ray at S=128, 128/S rays
// for shorter rays, ceil(S/128) chunks with a transmittance carry for longer ones).  For a tile:
//   front end  (128 threads, one sample each): ray march, NDC, 8-ch trilinear volume fetch,
//              3-view colour fetch, positional encoding            -> shared memory
//   MLP        (256 threads): ten GEMM passes over the 128-row tile, 8x8 register blocking,
//              weights streamed L2 -> smem in 32-row chunks with cp.async double buffering,
//              modulation / bias / activation fused into each pass epilogue
//   back end   alpha compositing in shared memory, one 16-byte result per ray to HBM.
// Front end and MLP are the fp32 forward tile (tile_fp32.cuh) the fine-tuning backward recomputes.
// No per-sample value ever goes to HBM unless the caller asks for the optional outputs.
//
// Replaces renderer.rendering (renderer.py:138-165) and callees; see include/mvsnerf_b200.h.
#include "tile_fp32.cuh"

namespace mvsn {

constexpr int SMEM_FLOATS = TILE_SMEM_FLOATS + TILE_M * 2;
constexpr size_t SMEM_BYTES = SMEM_FLOATS * sizeof(float);

template <bool FAST>
__global__ void __launch_bounds__(256, 1)
render_fp32_kernel(const SceneDev sc, const RenderIO io, const float* __restrict__ wts) {
    extern __shared__ __align__(16) float smem[];
    const TileSmem sm(smem);
    float* s_carry = sm.tail;                      // [8]: T carry, rgb/depth/acc partial sums (S > 128)

    const int tid = threadIdx.x;
    __shared__ Cams cams;
    load_cams(sc, &cams, tid);
    __syncthreads();
    const int N = io.N, S = io.S;
    const int R = S <= TILE_M ? TILE_M / S : 1;                 // rays per tile
    const int nchunks = S <= TILE_M ? 1 : (S + TILE_M - 1) / TILE_M;
    const int ngroups = (N + R - 1) / R;

    for (int grp = blockIdx.x; grp < ngroups; grp += gridDim.x) {
        for (int chunk = 0; chunk < nchunks; ++chunk) {
            int r_in = 0, s_idx = 0;
            bool valid = false;
            if (tid < TILE_M) {
                if (S <= TILE_M) { r_in = tid / S; s_idx = tid - r_in * S; valid = r_in < R; }
                else { r_in = 0; s_idx = chunk * TILE_M + tid; valid = s_idx < S; }
                valid = valid && grp * R + r_in < N;
                tile_front_end<FAST>(sc, cams, io, sm, tid, grp * R + r_in, s_idx, valid, NoRecord{});
            }
            __syncthreads();
            tile_mlp(sm, wts, tid, NoRecord{});
            if (tid < TILE_M) sm.sig[tid] = (1.f - sm.rgb[tid * 4 + 3]) + 1e-10f;   // sigma -> transmittance factor
            __syncthreads();

            // ------------------------------ compositing (renderer.py:65-92) ----------------
            if (tid < TILE_M && valid) {
                const int first = tid - (S <= TILE_M ? s_idx : tid);   // first row of this ray in the tile
                float T = (chunk == 0) ? 1.f : s_carry[0];
                for (int j = first; j < tid; ++j) T *= sm.sig[j];
                const float a = sm.rgb[tid * 4 + 3];
                const float w = a * T;
                const size_t si = (size_t)(grp * R + r_in) * S + s_idx;
                if (io.alpha) io.alpha[si] = a;
                if (io.weights) io.weights[si] = w;
                sm.z[tid] *= w;                                // depth contribution
                sm.rgb[tid * 4 + 3] = w;
            }
            __syncthreads();
            if (tid < R && grp * R + tid < N) {
                // one thread per ray sums its samples in order
                const int first = tid * (S <= TILE_M ? S : 0);
                const int cnt = S <= TILE_M ? S : min(TILE_M, S - chunk * TILE_M);
                float cr = 0.f, cg = 0.f, cb = 0.f, dp = 0.f, ac = 0.f, T = 1.f;
                if (chunk > 0) { T = s_carry[0]; cr = s_carry[1]; cg = s_carry[2]; cb = s_carry[3]; dp = s_carry[4]; ac = s_carry[5]; }
                for (int j = first; j < first + cnt; ++j) {
                    const float w = sm.rgb[j * 4 + 3];
                    cr = fmaf(w, sm.rgb[j * 4 + 0], cr); cg = fmaf(w, sm.rgb[j * 4 + 1], cg);
                    cb = fmaf(w, sm.rgb[j * 4 + 2], cb);
                    dp += sm.z[j]; ac += w; T *= sm.sig[j];
                }
                if (chunk + 1 < nchunks) {
                    s_carry[0] = T; s_carry[1] = cr; s_carry[2] = cg; s_carry[3] = cb; s_carry[4] = dp; s_carry[5] = ac;
                } else {
                    const int ray = grp * R + tid;
                    if (sc.white_bkgd) { const float bg = 1.f - ac; cr += bg; cg += bg; cb += bg; }
                    store_pixel(io, ray, cr, cg, cb, dp);
                }
            }
            __syncthreads();
        }
    }
}

int launch_render_fp32(const SceneDev& sc, const RenderIO& io, bool fast, const float* wts, cudaStream_t stream) {
    static bool attr_set[64] = {false};                   // once per device, not per launch
    int dev = 0;
    MVSN_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !attr_set[dev]) {
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_fp32_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_fp32_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
        if (dev < 64) attr_set[dev] = true;
    }
    const int R = io.S <= TILE_M ? TILE_M / io.S : 1;
    const int ngroups = (io.N + R - 1) / R;
    const int grid = ngroups < sm_count() ? ngroups : sm_count();
    if (grid <= 0) return MVSN_OK;
    if (fast) render_fp32_kernel<true><<<grid, 256, SMEM_BYTES, stream>>>(sc, io, wts);
    else      render_fp32_kernel<false><<<grid, 256, SMEM_BYTES, stream>>>(sc, io, wts);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

}  // namespace mvsn
