// K-C backward: the per-scene fine-tuning step of the fused render path as ONE kernel (SURVEY.md 8(f) row 2).
//
// Reference: train_mvs_nerf_finetuning_pl.py:140-189 -- `rendering(...)` under autograd, img2mse loss, Adam over the
// 22 MLP tensors (models.py:145-222) and RefVolume.feat_volume (models.py:935-950).  What autograd computes there
// with ~200 library launches per step is done here by
//
//   render_bwd_kernel      per tile of 128 samples: recompute the forward with the fp32 render kernel's own forward
//                          tile (tile_fp32.cuh; N_samples <= 128, so a tile holds whole rays and needs no chunk carry),
//                          reverse compositing scan, MLP dgrad + wgrad as tiled GEMMs, trilinear scatter-add of the
//                          8 volume-feature gradients into the channels-last volume gradient;
//   mlp_grad_reduce_kernel per-CTA private weight-gradient accumulators -> the 22 tensors in nn.Linear layout;
//   adam_*_kernel          fused Adam (torch.optim.Adam arithmetic) on the MLP tensors and on the volume.
//
// Data flow of a tile (one persistent CTA of 256 threads per SM, 7 tiles per CTA at 1024 rays x 128 samples):
//   * the forward recompute records (ScratchRecord) what the backward needs in a per-CTA scratch in global memory
//     (704 KB, L2 resident): the layer outputs TRANSPOSED (hT[n][r]) -- that is exactly the A operand of the wgrad GEMM
//     dW^T[k][n] = sum_r x^T[k][r] dpre[r][n], and the element-wise stage reads the same fragment shape from it;
//   * the pre-activation is not stored: h = relu(pre * mod) > 0  =>  pre = h / mod, and the sample does not
//     contribute where h == 0;
//   * every GEMM uses the forward kernel's tuned pattern: A row-major in shared memory, B streamed global -> shared
//     by cp.async.  dgrad:  A = dpre [r][n] (shared), B = W[n][k] (the nn.Linear layout itself);
//                   wgrad:  A = x^T (scratch -> shared), B = dpre [r][n] (scratch).  No shared-memory transposes.
//   * weight gradients accumulate in a per-CTA private buffer (plain read-modify-write, no atomics, deterministic);
//     the only atomics are the volume scatter (red.global.add.v4.f32, 16 per sample).
// Gradient inputs: d rgb (required, or a target image for the fused MSE loss), d depth, d weights, d alpha,
// d input_feat (optional) -- everything `rendering` returns is differentiable as in the reference.
//
// grad_mode MVSN_MLP_TC_HALF (mvsn_render_backward_tc) runs render_bwd_tc_kernel instead: the same tile with its
// dgrad / wgrad GEMMs on wgmma with fp16 operands; its schedule and numerics are described above the kernel.
// grad_mode MVSN_GRAD_TC_FULL (rays entries only) runs it with FULL = true: the forward recompute's MLP on wgmma too
// (tile_mlp_tc, described above it).
//
// mvsn_render_backward_deterministic runs either kernel with DET = true: the volume scatter and the fused loss are
// recorded instead of summed with float atomics, then summed in a fixed-point scatter and a fixed-order reduction
// (described above det_scatter_kernel), so every output is bit-reproducible.
//
// mvsn_render_backward_rays runs any of these with FAST = true: the front end marches the samples from the rays, as
// render_rays does, with stratified depths from a caller-drawn jitter (ray_z_jittered), instead of reading the
// per-sample arrays of ray_marcher / get_ndc_coordinate.
//
// mvsn_render_backward_rays_stop (FAST = true) and mvsn_render_backward_stop (FAST = false, the per-sample arrays) run
// the FP32 and TC_HALF kernels with STOP = true: early ray termination (described above StopTables).
#include <cfloat>

#include "tile_fp32.cuh"
#include "hopper.cuh"

namespace mvsn {

namespace bwd {
// per-CTA scratch (floats)
constexpr int S_PET   = 0;                        // [64][128]  peT[k][r]        (row 63 zero)
constexpr int S_FEATT = S_PET + 64 * 128;         // [64][128]  featT[k][r]      (rows >= 20 zero)
constexpr int S_MODT  = S_FEATT + 64 * 128;       // [128][128] modT[n][r]
constexpr int S_HT    = S_MODT + 128 * 128;       // 6 x [128][128] hT[l][n][r] = h_{l+1}
constexpr int S_FT    = S_HT + 6 * 128 * 128;     // [128][128] fT[k][r]  (feature_linear output)
constexpr int S_DPRE  = S_FT + 128 * 128;         // [128][128] row-major: B operand of the wgrad GEMMs
constexpr int S_DMOD  = S_DPRE + 128 * 128;       // [128][128] d modT[n][r] accumulator
constexpr int SCRATCH = S_DMOD + 128 * 128;
// per-CTA private gradient accumulators (floats); "T" = [k][n]
constexpr int G_W0T   = 0;                        // [64][128]
constexpr int G_W14T  = G_W0T + 64 * 128;         // 4 x [128][128]
constexpr int G_W5PET = G_W14T + 4 * 128 * 128;   // [64][128]
constexpr int G_W5HT  = G_W5PET + 64 * 128;       // [128][128]
constexpr int G_WBT   = G_W5HT + 128 * 128;       // [64][128]   (k < 20 used)
constexpr int G_WFT   = G_WBT + 64 * 128;         // [128][128]
constexpr int G_WVFT  = G_WFT + 128 * 128;        // [128 k][64 j]
constexpr int G_B     = G_WVFT + 128 * 64;        // b0..b5: 6 x [128]
constexpr int G_BB    = G_B + 6 * 128;
constexpr int G_BF    = G_BB + 128;
constexpr int G_WA    = G_BF + 128;
constexpr int G_BV    = G_WA + 128;               // [64]
constexpr int G_WVDT  = G_BV + 64;                // [4][64] (3 used)
constexpr int G_WR    = G_WVDT + 4 * 64;          // [4][64] (3 used)
constexpr int G_BR    = G_WR + 4 * 64;            // [4]: br[0..2], ba
constexpr int GRADS   = G_BR + 4;
// dgrad weight image (floats): B operands [n_out][k_in] of the dgrad GEMMs
constexpr int D_VF = 0;                           // views_linears.0.weight[:, :128]   [64][128]
constexpr int D_F  = D_VF + 64 * 128;             // feature_linear.weight             [128][128]
constexpr int D_5H = D_F + 128 * 128;             // pts_linears.5.weight[:, 63:]      [128][128]
constexpr int D_14 = D_5H + 128 * 128;            // pts_linears.1..4.weight           4 x [128][128]
constexpr int D_B  = D_14 + 4 * 128 * 128;        // pts_bias.weight                   [128][64] (k < 20)
constexpr int DGRAD = D_B + 128 * 64;
}  // namespace bwd

struct BwdIO {
    const float* g_rgb;      // [N,3]   (or null with `target`)
    const float* target;     // [N,3]   fused loss: g_rgb = 2 (rgb - target) / (3 N_total)
    float inv_count;         // 1 / (3 N_total)
    const float* g_depth;    // [N]     optional
    const float* g_weights;  // [N,S]   optional
    const float* g_alpha;    // [N,S]   optional
    const float* g_feat;     // [N,S,20] optional (only the 8 volume channels carry a gradient)
    float* dvol;             // [D,Hp,Wp,8] channels-last, accumulated atomically (null: the volume is frozen)
    float* scratch;          // n_ctas x bwd::SCRATCH
    float* grads;            // n_ctas x bwd::GRADS
    const float* wd;         // dgrad weight image
    float* rgb_out;          // [N,3] optional: the forward result of the recompute
    float* depth_out;        // [N]   optional
    float* loss;             // [1]   optional: += sum (rgb - target)^2 * inv_count
};

// What the DET = true kernels record instead of adding atomically (mvsn_render_backward_deterministic)
struct DetIO {
    float* rec;              // [N*S][8] each sample's 8 volume-feature gradients (null: the volume is frozen)
    float* loss_terms;       // [N] each ray's loss term (with bw.loss)
    unsigned* amax;          // [2] max |g| over the finite recorded values (float bits), and a non-finite flag
};

// What the STOP = true kernels (mvsn_render_backward_rays_stop, mvsn_render_backward_stop) take besides
struct StopIO {
    float t_stop;                    // sample j of a ray is live iff its transmittance T_j >= t_stop
    int* live;                       // [N] live samples per ray (the caller's live_samples, or the workspace)
    int2* list;                      // per CTA: list_cap (ray, live samples) entries deferred to phase B
    int list_cap;
    unsigned long long* tiles_done;  // [3] += tiles back-propagated immediately, deferred, packed (may be null)
};

namespace {

// fragment <-> memory helpers of the backward (fragment layout: frag_row / frag_col in tile_fp32.cuh)
// transposed store: dstT[col][row] with 128-float rows (global scratch)
__device__ __forceinline__ void frag_store_T(const float (&acc)[8][8], float* dstT, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
        float* p = dstT + frag_col(tx, n) * 128 + ty * 4;
        *reinterpret_cast<float4*>(p) = make_float4(acc[0][n], acc[1][n], acc[2][n], acc[3][n]);
        *reinterpret_cast<float4*>(p + 64) = make_float4(acc[4][n], acc[5][n], acc[6][n], acc[7][n]);
    }
}
__device__ __forceinline__ void frag_load_T(float (&v)[8][8], const float* srcT, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
        const float* p = srcT + frag_col(tx, n) * 128 + ty * 4;
        const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 64);
        v[0][n] = a.x; v[1][n] = a.y; v[2][n] = a.z; v[3][n] = a.w;
        v[4][n] = b.x; v[5][n] = b.y; v[6][n] = b.z; v[7][n] = b.w;
    }
}
// private accumulator += fragment, row-major [rows][ld] in global memory
template <int MR, int NT>
__device__ __forceinline__ void frag_accumulate(const float (&acc)[MR][NT], float* dst, int ld, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
#pragma unroll
    for (int r = 0; r < MR; ++r) {
        float* p = dst + frag_row(ty, r) * ld + tx * 4;
        float4 a = *reinterpret_cast<float4*>(p);
        a.x += acc[r][0]; a.y += acc[r][1]; a.z += acc[r][2]; a.w += acc[r][3];
        *reinterpret_cast<float4*>(p) = a;
        if constexpr (NT == 8) {
            float4 b = *reinterpret_cast<float4*>(p + 64);
            b.x += acc[r][4]; b.y += acc[r][5]; b.z += acc[r][6]; b.w += acc[r][7];
            *reinterpret_cast<float4*>(p + 64) = b;
        }
    }
}
// [rows][128] dense global -> shared [rows][H_LD]
__device__ __forceinline__ void stage_T(float* s_dst, const float* g_src, int rows, int tid) {
    for (int i = tid; i < rows * 32; i += 256) {
        const int r = i >> 5, c4 = i & 31;
        cp_async16(s_dst + r * H_LD + c4 * 4, g_src + r * 128 + c4 * 4);
    }
    cp_async_commit();
}
// column sums of a row-major shared tile [128][ld], columns [0, ncols): thread c accumulates into dst[c]
__device__ __forceinline__ void colsum_accumulate(const float* s_src, int ld, int ncols, float* dst, int tid) {
    if (tid < ncols) {
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < TILE_M; ++r) s += s_src[r * ld + tid];
        dst[tid] += s;
    }
}

// What the backward keeps of the forward, in the CTA's scratch: the layer inputs and outputs transposed
struct ScratchRecord {
    float* scr;
    __device__ __forceinline__ void pe(int row, int k, float v) const { scr[bwd::S_PET + k * 128 + row] = v; }
    __device__ __forceinline__ void feat(int row, int k, float v) const { scr[bwd::S_FEATT + k * 128 + row] = v; }
    __device__ __forceinline__ void mod(const float (&acc)[8][8], int tid) const { frag_store_T(acc, scr + bwd::S_MODT, tid); }
    __device__ __forceinline__ void hidden(int l, const float (&acc)[8][8], int tid) const {
        frag_store_T(acc, scr + bwd::S_HT + l * 16384, tid);
    }
    __device__ __forceinline__ void feature(const float (&acc)[8][8], int tid) const { frag_store_T(acc, scr + bwd::S_FT, tid); }
};

constexpr int BWD_SMEM_FLOATS = TILE_SMEM_FLOATS + TILE_M * 18;
constexpr size_t BWD_SMEM_BYTES = BWD_SMEM_FLOATS * sizeof(float);
static_assert(TILE_M * PE_LD >= 64 * H_LD, "peT staging [64][H_LD] must fit in the positional-encoding region");

// ---- early ray termination (STOP = true, mvsn_render_backward_rays_stop / mvsn_render_backward_stop) ---------------
// Sample j of a ray is live iff T_j >= t_stop (T_0 = 1, T_{j+1} = T_j ((1 - alpha_j) + 1e-10), the scan's fp32 order);
// T never increases, so the live samples are a prefix of length L.  The kernel differentiates exactly the truncated
// render sum_{j<L} w_j c_j: dead samples get s_g = 0 and no volume scatter.  Two phases in the persistent launch:
//   A  the CTA's static groups, as the other kernels take them.  After the forward scan the tile is back-propagated
//      at once (dead rows zero: every GEMM, column sum and scatter is linear in s_g) unless some of its samples are
//      dead and fewer than TILE_M / 2 rows are live; then its rays (ray, L) are appended to the CTA's list instead.
//   B  the CTA's listed rays, in list order and whole, packed into 128-row tiles, recomputed and back-propagated.
// The tile's rows and rays come from tables in shared memory behind the backward's own (StopTables); the forward
// tile, the GEMMs and the heads do not care which rows they hold.  A sample's forward is its own row's (fp32, row-
// independent), so its alpha, and the ray's L, are the same in both phases; rgb / depth / the loss are written in
// phase A only.
namespace stopt {
constexpr int ROW_SLOT = 0;                  // [128] row -> ray slot of the tile, -1: empty row
constexpr int ROW_S    = ROW_SLOT + TILE_M;  // [128] row -> sample index in its ray
constexpr int RAY      = ROW_S + TILE_M;     // [128] slot -> ray (-1: past N)
constexpr int FIRST    = RAY + TILE_M;       // [128] slot -> first row
constexpr int LEN      = FIRST + TILE_M;     // [128] slot -> rows (after the scan: live samples)
constexpr int MISC     = LEN + TILE_M;
enum { N_RAYS, N_ROWS, LIVE_ROWS, PHASE_B, N_LIST, CURSOR, N_IMM, N_DEF, N_PACKED, N_MISC };
constexpr int INTS     = MISC + N_MISC;
}  // namespace stopt
constexpr size_t STOP_SMEM_BYTES = stopt::INTS * sizeof(int);

struct StopTables {
    int* t;
    __device__ __forceinline__ explicit StopTables(float* smem) : t(reinterpret_cast<int*>(smem + BWD_SMEM_FLOATS)) {}
    __device__ __forceinline__ int& misc(int i) const { return t[stopt::MISC + i]; }
};

// phase A: group grp in the standard mapping (slot r = ray grp * R + r, rows [r S, r S + S))
__device__ __forceinline__ void stop_plan_group(const StopTables& st, int grp, int R, int S, int N, int tid) {
    if (tid < TILE_M) {
        const int r_in = tid / S;
        st.t[stopt::ROW_SLOT + tid] = r_in < R && grp * R + r_in < N ? r_in : -1;
        st.t[stopt::ROW_S + tid] = tid - r_in * S;
    }
    if (tid < R) {
        const int ray = grp * R + tid;
        st.t[stopt::RAY + tid] = ray < N ? ray : -1;
        st.t[stopt::FIRST + tid] = tid * S;
        st.t[stopt::LEN + tid] = S;
    }
    if (tid == 0) { st.misc(stopt::N_RAYS) = R; st.misc(stopt::N_ROWS) = R * S; st.misc(stopt::LIVE_ROWS) = 0; }
}

// phase B, one thread: the next packed tile from the CTA's list (N_RAYS = 0: the list is done)
__device__ __forceinline__ void stop_pack_tile(const StopTables& st, const int2* list) {
    int c = st.misc(stopt::CURSOR), rows = 0, k = 0;
    const int n = st.misc(stopt::N_LIST);
    for (; c < n; ++c, ++k) {
        const int2 e = list[c];                              // e.y >= 1: T_0 = 1 >= t_stop
        if (rows + e.y > TILE_M) break;
        st.t[stopt::RAY + k] = e.x; st.t[stopt::FIRST + k] = rows; st.t[stopt::LEN + k] = e.y;
        for (int s = 0; s < e.y; ++s) { st.t[stopt::ROW_SLOT + rows + s] = k; st.t[stopt::ROW_S + rows + s] = s; }
        rows += e.y;
    }
    for (int r = rows; r < TILE_M; ++r) { st.t[stopt::ROW_SLOT + r] = -1; st.t[stopt::ROW_S + r] = 0; }
    st.misc(stopt::CURSOR) = c; st.misc(stopt::N_RAYS) = k; st.misc(stopt::N_ROWS) = rows;
    st.misc(stopt::LIVE_ROWS) = 0; st.misc(stopt::PHASE_B) = 1;
    if (k) ++st.misc(stopt::N_PACKED);
}

// Top of a tile: the tables of phase A's group grp, or of phase B's next packed tile.  False: nothing left.
__device__ __forceinline__ bool stop_next_tile(float* smem, const StopIO& stop, int grp, int ngroups, int R, int S, int N,
                                               int tid) {
    const StopTables st(smem);
    if (grp < ngroups) stop_plan_group(st, grp, R, S, N, tid);
    else if (tid == 0) stop_pack_tile(st, stop.list + (size_t)blockIdx.x * stop.list_cap);
    __syncthreads();
    return st.misc(stopt::N_RAYS) != 0;
}

// Row tid of the tile (tid < TILE_M): its ray and sample; false for an empty row
__device__ __forceinline__ bool stop_row(float* smem, int tid, int& ray, int& s_idx) {
    const StopTables st(smem);
    const int slot = st.t[stopt::ROW_SLOT + tid];
    s_idx = st.t[stopt::ROW_S + tid];
    ray = slot >= 0 ? st.t[stopt::RAY + slot] : 0;
    return slot >= 0;
}

// After the forward scan: whether row tid holds a live sample (the rows the volume scatter takes)
__device__ __forceinline__ bool stop_row_live(float* smem, int tid) {
    const StopTables st(smem);
    const int slot = st.t[stopt::ROW_SLOT + tid];
    return slot >= 0 && st.t[stopt::ROW_S + tid] < st.t[stopt::LEN + slot];
}

// Phase A, after the forward scan and a barrier: defer the tile (append its rays to the CTA's list) or back-propagate
// it now.  A tile none of whose samples is dead is never deferred, so t_stop = 0 does exactly the work of the kernels
// without STOP.  Ends with a barrier (every thread has read the counters thread 0 then updates).
__device__ __forceinline__ bool stop_defer(float* smem, const StopIO& stop, int grp, int ngroups, int R, int S, int N,
                                           int tid) {
    const StopTables st(smem);
    if (grp >= ngroups) return false;                          // a packed tile (phase B)
    const int nvalid = min(R, N - grp * R), live = st.misc(stopt::LIVE_ROWS);
    const bool defer = live < nvalid * S && 2 * live < TILE_M;
    if (defer && tid < nvalid)
        stop.list[(size_t)blockIdx.x * stop.list_cap + st.misc(stopt::N_LIST) + tid] =
            make_int2(st.t[stopt::RAY + tid], st.t[stopt::LEN + tid]);
    __syncthreads();
    if (tid == 0) {
        if (defer) { st.misc(stopt::N_LIST) += nvalid; ++st.misc(stopt::N_DEF); }
        else ++st.misc(stopt::N_IMM);
    }
    return defer;
}

__device__ __forceinline__ void stop_init(float* smem, int tid) {
    if (tid < stopt::N_MISC) StopTables(smem).misc(tid) = 0;
}

__device__ __forceinline__ void stop_finish(float* smem, const StopIO& stop, int tid) {
    const StopTables st(smem);
    if (tid == 0 && stop.tiles_done) {
        atomicAdd(stop.tiles_done, (unsigned long long)st.misc(stopt::N_IMM));
        atomicAdd(stop.tiles_done + 1, (unsigned long long)st.misc(stopt::N_DEF));
        atomicAdd(stop.tiles_done + 2, (unsigned long long)st.misc(stopt::N_PACKED));
    }
}

// Compositing of a tile, forward and reverse scan, one thread per ray (renderer.py:65-92).  Writes rgb_out /
// depth_out / the fused loss, s_T (transmittance in front of each sample) and s_g (d rgb_pre, d sigma_pre per row).
// f_j = 1 - alpha_j + 1e-10, T_{j+1} = T_j f_j, w_j = alpha_j T_j.
// d alpha_j = T_j (d w_j - B_j),  B_{j-1} = d w_j alpha_j + f_j B_j  (no division by f_j).
// DET: the ray's loss term goes to det.loss_terms[ray] instead of being added to bw.loss.
// STOP: the rays and rows come from the StopTables; the forward stops at the first dead sample (T_j < t_stop), the
// ray's live count L goes to the table (LEN) and, in phase A, to stop->live; the dead rows get s_g = 0; rgb_out /
// depth_out / the loss are written in phase A only.
template <bool DET, bool STOP = false>
__device__ __forceinline__ void composite_scan(const SceneDev& sc, const BwdIO& bw, const TileSmem& sm, float* s_T, float* s_g,
                                               int grp, int R, int S, int N, int tid, const DetIO& det,
                                               const StopIO* stop = nullptr, float* smem = nullptr) {
    int nrays = R, nrows = R * S;
    bool emit = true;
    if constexpr (STOP) {
        const StopTables st(smem);
        nrays = st.misc(stopt::N_RAYS); nrows = st.misc(stopt::N_ROWS); emit = st.misc(stopt::PHASE_B) == 0;
    }
    if (tid < nrays) {
        int ray = grp * R + tid, first = tid * S, len = S;
        bool ok = ray < N;
        if constexpr (STOP) {
            const StopTables st(smem);
            ray = st.t[stopt::RAY + tid]; first = st.t[stopt::FIRST + tid]; len = st.t[stopt::LEN + tid]; ok = ray >= 0;
        }
        if (ok) {
            float cr = 0.f, cg = 0.f, cb = 0.f, dp = 0.f, ac = 0.f, T = 1.f;
            int end = first + len;
            for (int j = first; j < first + len; ++j) {
                if constexpr (STOP) { if (T < stop->t_stop) { end = j; break; } }
                const float a = sm.rgb[j * 4 + 3], w = a * T;
                s_T[j] = T;
                cr = fmaf(w, sm.rgb[j * 4 + 0], cr); cg = fmaf(w, sm.rgb[j * 4 + 1], cg); cb = fmaf(w, sm.rgb[j * 4 + 2], cb);
                dp = fmaf(w, sm.z[j], dp); ac += w;
                T *= (1.f - a) + 1e-10f;
            }
            if constexpr (STOP) {
                const StopTables st(smem);
                const int L = end - first;
                for (int j = end; j < first + len; ++j) { s_g[j * 4] = s_g[j * 4 + 1] = s_g[j * 4 + 2] = s_g[j * 4 + 3] = 0.f; }
                st.t[stopt::LEN + tid] = L;
                if (emit) stop->live[ray] = L;
                atomicAdd(&st.misc(stopt::LIVE_ROWS), L);
            }
            if (sc.white_bkgd) { const float bg = 1.f - ac; cr += bg; cg += bg; cb += bg; }
            if (emit && bw.rgb_out) { bw.rgb_out[(size_t)ray * 3] = cr; bw.rgb_out[(size_t)ray * 3 + 1] = cg; bw.rgb_out[(size_t)ray * 3 + 2] = cb; }
            if (emit && bw.depth_out) bw.depth_out[ray] = dp;
            float g0, g1, g2;
            if (bw.target) {                     // fused img2mse (utils.py: mean((rgb - target)^2))
                const float e0 = cr - __ldg(bw.target + (size_t)ray * 3), e1 = cg - __ldg(bw.target + (size_t)ray * 3 + 1),
                            e2 = cb - __ldg(bw.target + (size_t)ray * 3 + 2);
                g0 = 2.f * e0 * bw.inv_count; g1 = 2.f * e1 * bw.inv_count; g2 = 2.f * e2 * bw.inv_count;
                if (emit && bw.loss) {
                    if constexpr (DET) det.loss_terms[ray] = (e0 * e0 + e1 * e1 + e2 * e2) * bw.inv_count;
                    else               atomicAdd(bw.loss, (e0 * e0 + e1 * e1 + e2 * e2) * bw.inv_count);
                }
            } else {
                g0 = __ldg(bw.g_rgb + (size_t)ray * 3); g1 = __ldg(bw.g_rgb + (size_t)ray * 3 + 1); g2 = __ldg(bw.g_rgb + (size_t)ray * 3 + 2);
            }
            const float gd = bw.g_depth ? __ldg(bw.g_depth + ray) : 0.f;
            const float gbg = sc.white_bkgd ? (g0 + g1 + g2) : 0.f;
            float B = 0.f;
            for (int j = end - 1; j >= first; --j) {
                const size_t sj = (size_t)ray * S + (j - first);
                const float a = sm.rgb[j * 4 + 3], Tj = s_T[j], w = a * Tj;
                const float c0 = sm.rgb[j * 4], c1 = sm.rgb[j * 4 + 1], c2 = sm.rgb[j * 4 + 2];
                float dw = g0 * c0 + g1 * c1 + g2 * c2 + gd * sm.z[j] - gbg;
                if (bw.g_weights) dw += __ldg(bw.g_weights + sj);
                float da = Tj * (dw - B);
                if (bw.g_alpha) da += __ldg(bw.g_alpha + sj);
                B = fmaf(((1.f - a) + 1e-10f), B, dw * a);
                s_g[j * 4 + 0] = w * g0 * c0 * (1.f - c0);
                s_g[j * 4 + 1] = w * g1 * c1 * (1.f - c1);
                s_g[j * 4 + 2] = w * g2 * c2 * (1.f - c2);
                s_g[j * 4 + 3] = sm.sig[j] > 0.f ? da * (1.f - a) : 0.f;
            }
        } else {
            for (int j = first; j < first + len; ++j) { s_g[j * 4] = s_g[j * 4 + 1] = s_g[j * 4 + 2] = s_g[j * 4 + 3] = 0.f; }
        }
    }
    if (tid >= nrows && tid < TILE_M) { s_g[tid * 4] = s_g[tid * 4 + 1] = s_g[tid * 4 + 2] = s_g[tid * 4 + 3] = 0.f; }
}

// Element-wise stage of trunk layer l on the thread's fragment: acc = d h_{l+1}  ->  d g = acc * (h > 0) ;
// d pre = d g * mod (left in acc) ; d mod += d g * pre, pre = h / mod (accumulated transposed in the scratch)
__device__ __forceinline__ void trunk_elementwise(float (&acc)[8][8], float* scr, int l, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
    const float* hT = scr + bwd::S_HT + l * 16384;
    const float* mT = scr + bwd::S_MODT;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
        const int col = frag_col(tx, n);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const float4 h4 = *reinterpret_cast<const float4*>(hT + col * 128 + half * 64 + ty * 4);
            const float4 m4 = *reinterpret_cast<const float4*>(mT + col * 128 + half * 64 + ty * 4);
            const float hh[4] = {h4.x, h4.y, h4.z, h4.w}, mm[4] = {m4.x, m4.y, m4.z, m4.w};
            float dm[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = half * 4 + i;
                const bool on = hh[i] > 0.f;
                const float dg = on ? acc[r][n] : 0.f;
                acc[r][n] = dg * mm[i];
                dm[i] = on ? dg * __fdiv_rn(hh[i], mm[i]) : 0.f;
            }
            float4* dmod = reinterpret_cast<float4*>(scr + bwd::S_DMOD + col * 128 + half * 64 + ty * 4);
            float4 o = make_float4(dm[0], dm[1], dm[2], dm[3]);
            if (l != 5) { const float4 p = *dmod; o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w; }
            *dmod = o;
        }
    }
}

// Trilinear scatter of row `tid`'s 8 volume-feature gradients (s_df, plus d input_feat) into the channels-last volume
// gradient: the transpose of utils.index_point_feature (utils.py:357-383), with the same corner weights.
// DET: the 8 gradients are recorded to det.rec[si] and folded into det.amax (max |g| over the finite values, as float
// bits with an integer atomicMax, so the result does not depend on the order; any non-finite value sets amax[1]);
// det_scatter_kernel scatters them afterwards.  The caller is divergent (valid rows only), hence __activemask.
// The sample's NDC: io.ndc[si], or (FAST: marched in the kernel) rows 0..2 of the recorded positional encoding peT in the
// CTA's scratch -- the front end's own values, so the scatter hits exactly the corners the forward sampled.
template <bool DET, bool FAST>
__device__ __forceinline__ void volume_scatter(const SceneDev& sc, const RenderIO& io, const BwdIO& bw, const float* s_df,
                                               size_t si, int tid, const DetIO& det, const float* scr) {
    float g8[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) g8[c] = s_df[tid * 8 + c];
    if (bw.g_feat) {
#pragma unroll
        for (int c = 0; c < 8; ++c) g8[c] += __ldg(bw.g_feat + si * 20 + c);
    }
    if constexpr (DET) {
        float4* r = reinterpret_cast<float4*>(det.rec + si * 8);
        r[0] = make_float4(g8[0], g8[1], g8[2], g8[3]);
        r[1] = make_float4(g8[4], g8[5], g8[6], g8[7]);
        float m = 0.f;
        unsigned nonfinite = 0u;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float a = fabsf(g8[c]);
            if (a <= FLT_MAX) m = fmaxf(m, a); else nonfinite = 1u;
        }
        const unsigned mask = __activemask();
        const unsigned mb = __reduce_max_sync(mask, __float_as_uint(m)), nf = __reduce_or_sync(mask, nonfinite);
        if ((tid & 31) == __ffs(mask) - 1) {
            if (mb) atomicMax(det.amax, mb);
            if (nf) atomicOr(det.amax + 1, nf);
        }
        return;
    }
    Trilinear t;
    if constexpr (FAST) t = trilinear_corners(sc, scr[bwd::S_PET + tid], scr[bwd::S_PET + 128 + tid], scr[bwd::S_PET + 256 + tid]);
    else t = trilinear_corners(sc, __ldg(io.ndc + si * 3), __ldg(io.ndc + si * 3 + 1), __ldg(io.ndc + si * 3 + 2));
    const int W = sc.Wp, H = sc.Hp, D = sc.D;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int x = t.x0 + (c & 1), y = t.y0 + ((c >> 1) & 1), z = t.z0 + (c >> 2);
        if ((unsigned)x >= (unsigned)W || (unsigned)y >= (unsigned)H || (unsigned)z >= (unsigned)D) continue;   // zeros padding
        const float wgt = t.wx[c & 1] * t.wy[(c >> 1) & 1] * t.wz[c >> 2];
        float4* p = reinterpret_cast<float4*>(bw.dvol + (((size_t)z * H + y) * W + x) * 8);
        atomicAdd(p, make_float4(g8[0] * wgt, g8[1] * wgt, g8[2] * wgt, g8[3] * wgt));
        atomicAdd(p + 1, make_float4(g8[4] * wgt, g8[5] * wgt, g8[6] * wgt, g8[7] * wgt));
    }
}

// FAST: the front end marches the samples from io.rays / io.t_steps (stratified by `jitter` [N,S] unless NULL) instead of
// reading io.pts / io.ndc / io.z / io.dirs (mvsn_render_backward_rays); `jitter` is unused otherwise.
// STOP: early ray termination at stop.t_stop, in two phases (described above StopTables); the launch adds
// STOP_SMEM_BYTES of dynamic shared memory for the tables.  `stop` is unused otherwise.
template <bool DET, bool FAST, bool STOP = false>
__global__ void __launch_bounds__(256, 1)
render_bwd_kernel(const SceneDev sc, const RenderIO io, const BwdIO bw, const float* __restrict__ wts, const DetIO det,
                  const float* __restrict__ jitter, const StopIO stop) {
    extern __shared__ __align__(16) float smem[];
    const TileSmem sm(smem);                       // backward: sm.pe holds peT as [64][H_LD]; sm.h, sm.mod the A operands
    float* s_T    = sm.tail;                       // [128] transmittance in front of the sample
    float* s_g    = s_T + TILE_M;                  // [128][4] d rgb_pre (3), d sigma_pre
    float* s_df   = s_g + TILE_M * 4;              // [128][8] d volume features ; [128][4] spare
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    __shared__ Cams cams;
    load_cams(sc, &cams, tid);

    float* scr = bw.scratch + (size_t)blockIdx.x * bwd::SCRATCH;
    float* G = bw.grads + (size_t)blockIdx.x * bwd::GRADS;
    for (int i = tid; i < bwd::GRADS; i += 256) G[i] = 0.f;
    for (int i = tid; i < 32 * 128; i += 256) scr[bwd::S_FEATT + 32 * 128 + i] = 0.f;      // featT rows 32..63 stay zero
    if constexpr (STOP) stop_init(smem, tid);
    __syncthreads();

    const int N = io.N, S = io.S;
    const int R = TILE_M / S;                                   // rays per tile (S <= 128, checked by the launcher)
    const int ngroups = (N + R - 1) / R;

    // STOP: phase A's groups, then phase B's packed tiles (grp >= ngroups) until the CTA's list is done
    for (int grp = blockIdx.x; STOP || grp < ngroups; grp += gridDim.x) {
        if constexpr (STOP) { if (!stop_next_tile(smem, stop, grp, ngroups, R, S, N, tid)) break; }
        // =============================== forward recompute ===========================================
        bool valid = false;
        size_t si = 0;
        if (tid < TILE_M) {
            if constexpr (STOP) {
                int ray, s_idx;
                valid = stop_row(smem, tid, ray, s_idx);
                si = (size_t)ray * S + s_idx;
                tile_front_end<FAST>(sc, cams, io, sm, tid, ray, s_idx, valid, ScratchRecord{scr}, jitter);
            } else {
                const int r_in = tid / S, s_idx = tid - r_in * S, ray = grp * R + r_in;
                valid = r_in < R && ray < N;
                si = (size_t)ray * S + s_idx;
                tile_front_end<FAST>(sc, cams, io, sm, tid, ray, s_idx, valid, ScratchRecord{scr}, jitter);
            }
        }
        __syncthreads();
        tile_mlp(sm, wts, tid, ScratchRecord{scr});
        __syncthreads();

        // =============================== compositing: forward + reverse scan ===========================
        composite_scan<DET, STOP>(sc, bw, sm, s_T, s_g, grp, R, S, N, tid, det, &stop, smem);
        if constexpr (STOP) {
            __syncthreads();                                    // every ray's live count
            if (stop_defer(smem, stop, grp, ngroups, R, S, N, tid)) continue;
        }
        stage_T(sm.pe, scr + bwd::S_PET, 64, tid);             // peT -> shared (used by the layer-5 and layer-0 wgrads)
        __syncthreads();

        // =============================== backward through the heads =================================
        // rgb_linear: d Wr, d br, d ba (small reductions over the 128 rows), d hv_pre
        if (tid < 64) {
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
            for (int r = 0; r < TILE_M; ++r) {
                const float h = sm.mod[r * HV_LD + tid];
                a0 = fmaf(s_g[r * 4], h, a0); a1 = fmaf(s_g[r * 4 + 1], h, a1); a2 = fmaf(s_g[r * 4 + 2], h, a2);
            }
            G[bwd::G_WR + tid] += a0; G[bwd::G_WR + 64 + tid] += a1; G[bwd::G_WR + 128 + tid] += a2;
        } else if (tid < 68) {
            const int c = tid - 64;
            float a = 0.f;
            for (int r = 0; r < TILE_M; ++r) a += s_g[r * 4 + c];
            G[bwd::G_BR + c] += a;                             // c == 3: d ba = sum d sigma_pre
        }
        {
            // d hv_pre[r][j] = (hv > 0) * sum_c d rgb_pre[r][c] Wr[c][j]   -> sm.h (A, lda H_LD) and scratch [128][64] (B)
            const float4 w0 = __ldg(reinterpret_cast<const float4*>(wts + w32::WR + tx * 4));
            const float4 w1 = __ldg(reinterpret_cast<const float4*>(wts + w32::WR + 64 + tx * 4));
            const float4 w2 = __ldg(reinterpret_cast<const float4*>(wts + w32::WR + 128 + tx * 4));
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const int row = frag_row(ty, r);
                const float d0 = s_g[row * 4], d1 = s_g[row * 4 + 1], d2 = s_g[row * 4 + 2];
                const float4 hv = *reinterpret_cast<const float4*>(sm.mod + row * HV_LD + tx * 4);
                float4 o;
                o.x = hv.x > 0.f ? fmaf(d2, w2.x, fmaf(d1, w1.x, d0 * w0.x)) : 0.f;
                o.y = hv.y > 0.f ? fmaf(d2, w2.y, fmaf(d1, w1.y, d0 * w0.y)) : 0.f;
                o.z = hv.z > 0.f ? fmaf(d2, w2.z, fmaf(d1, w1.z, d0 * w0.z)) : 0.f;
                o.w = hv.w > 0.f ? fmaf(d2, w2.w, fmaf(d1, w1.w, d0 * w0.w)) : 0.f;
                *reinterpret_cast<float4*>(sm.h + row * H_LD + tx * 4) = o;
                *reinterpret_cast<float4*>(scr + bwd::S_DPRE + row * 64 + tx * 4) = o;
            }
        }
        __syncthreads();                                        // hv (sm.mod) no longer needed; d hv_pre complete
        stage_T(sm.mod, scr + bwd::S_FT, 128, tid);              // fT -> A operand of the views wgrad
        if (tid < 64) {                                         // d bv, d Wv[:, 128:131]^T
            float sb = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f;
            for (int r = 0; r < TILE_M; ++r) {
                const float d = sm.h[r * H_LD + tid];
                sb += d; s0 = fmaf(sm.dir[r * 4], d, s0); s1 = fmaf(sm.dir[r * 4 + 1], d, s1); s2 = fmaf(sm.dir[r * 4 + 2], d, s2);
            }
            G[bwd::G_BV + tid] += sb;
            G[bwd::G_WVDT + tid] += s0; G[bwd::G_WVDT + 64 + tid] += s1; G[bwd::G_WVDT + 128 + tid] += s2;
        }
        cp_async_wait<0>();
        __syncthreads();
        {
            float acc[8][4];                                    // d Wv_f^T[k][j] = sum_r fT[k][r] d hv_pre[r][j]
            zero_acc(acc);
            gemm_pass<64>(acc, sm.mod, H_LD, 128, scr + bwd::S_DPRE, sm.w, tid);
            frag_accumulate(acc, G + bwd::G_WVFT, 64, tid);
        }
        float acc[8][8];
        zero_acc(acc);                                          // d f[r][k] = sum_j d hv_pre[r][j] Wv[j][k]
        gemm_pass<128>(acc, sm.h, H_LD, 64, bw.wd + bwd::D_VF, sm.w, tid);
        frag_store_rm(acc, sm.h, H_LD, tid);
        frag_store_rm(acc, scr + bwd::S_DPRE, 128, tid);
        __syncthreads();
        stage_T(sm.mod, scr + bwd::S_HT + 5 * 16384, 128, tid);  // h6T
        colsum_accumulate(sm.h, H_LD, 128, G + bwd::G_BF, tid);  // d bf
        cp_async_wait<0>();
        __syncthreads();
        zero_acc(acc);                                          // d Wf^T[k][n] = sum_r h6T[k][r] d f[r][n]
        gemm_pass<128>(acc, sm.mod, H_LD, 128, scr + bwd::S_DPRE, sm.w, tid);
        frag_accumulate(acc, G + bwd::G_WFT, 128, tid);
        if (tid < TILE_M) {                                     // d wa[k] = sum_r d sigma_pre[r] h6T[k][r]
            float s = 0.f;
            for (int r = 0; r < TILE_M; ++r) s = fmaf(s_g[r * 4 + 3], sm.mod[tid * H_LD + r], s);
            G[bwd::G_WA + tid] += s;
        }
        zero_acc(acc);                                          // d h6 = d f Wf + d sigma_pre (x) wa
        gemm_pass<128>(acc, sm.h, H_LD, 128, bw.wd + bwd::D_F, sm.w, tid);
        {
            const float4 al = __ldg(reinterpret_cast<const float4*>(wts + w32::WA + tx * 4));
            const float4 ah = __ldg(reinterpret_cast<const float4*>(wts + w32::WA + 64 + tx * 4));
            const float wa[8] = {al.x, al.y, al.z, al.w, ah.x, ah.y, ah.z, ah.w};
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float ds = s_g[frag_row(ty, r) * 4 + 3];
#pragma unroll
                for (int n = 0; n < 8; ++n) acc[r][n] = fmaf(ds, wa[n], acc[r][n]);
            }
        }

        // =============================== trunk, layers 5..0 ==========================================
#pragma unroll 1
        for (int l = 5; l >= 0; --l) {
            // element-wise: acc = d h_{l+1}  ->  d g = acc * (h > 0) ; d pre = d g * mod ; d mod += d g * pre, pre = h / mod
            trunk_elementwise(acc, scr, l, tid);
            frag_store_rm(acc, sm.h, H_LD, tid);
            frag_store_rm(acc, scr + bwd::S_DPRE, 128, tid);
            __syncthreads();
            if (l >= 1) stage_T(sm.mod, scr + bwd::S_HT + (l - 1) * 16384, 128, tid);      // x_l^T = h_l^T
            colsum_accumulate(sm.h, H_LD, 128, G + bwd::G_B + l * 128, tid);                // d b_l
            cp_async_wait<0>();
            __syncthreads();
            if (l >= 1) {                                       // d W_l^T[k][n] = sum_r h_l^T[k][r] d pre[r][n]
                zero_acc(acc);
                gemm_pass<128>(acc, sm.mod, H_LD, 128, scr + bwd::S_DPRE, sm.w, tid);
                frag_accumulate(acc, G + (l == 5 ? bwd::G_W5HT : bwd::G_W14T + (l - 1) * 16384), 128, tid);
            }
            if (l == 5 || l == 0) {                             // positional-encoding part: 64-row A
                float a4[4][8];
                zero_acc(a4);
                gemm_pass<128>(a4, sm.pe, H_LD, 128, scr + bwd::S_DPRE, sm.w, tid);
                frag_accumulate(a4, G + (l == 5 ? bwd::G_W5PET : bwd::G_W0T), 128, tid);
            }
            if (l >= 1) {                                       // d h_l = d pre W_l (h part)
                zero_acc(acc);
                gemm_pass<128>(acc, sm.h, H_LD, 128, bw.wd + (l == 5 ? bwd::D_5H : bwd::D_14 + (l - 1) * 16384), sm.w, tid);
            }
        }
        // =============================== modulation branch: pts_bias ==================================
        // d mod is complete in scratch (transposed): bring it to row-major -- A operand of d feat (shared), B operand of d Wb
        frag_load_T(acc, scr + bwd::S_DMOD, tid);
        frag_store_rm(acc, sm.h, H_LD, tid);
        frag_store_rm(acc, scr + bwd::S_DPRE, 128, tid);
        stage_T(sm.mod, scr + bwd::S_FEATT, 64, tid);
        cp_async_wait<0>();
        __syncthreads();
        colsum_accumulate(sm.h, H_LD, 128, G + bwd::G_BB, tid);
        {
            float a4[4][8];                                     // d Wb^T[k][n] = sum_r featT[k][r] d mod[r][n]
            zero_acc(a4);
            gemm_pass<128>(a4, sm.mod, H_LD, 128, scr + bwd::S_DPRE, sm.w, tid);
            frag_accumulate(a4, G + bwd::G_WBT, 128, tid);
        }
        if (bw.dvol) {
            float a[8][4];                                      // d feat[r][k] = sum_n d mod[r][n] Wb[n][k]
            zero_acc(a);
            gemm_pass<64>(a, sm.h, H_LD, 128, bw.wd + bwd::D_B, sm.w, tid);
            if (tx < 2) {
#pragma unroll
                for (int r = 0; r < 8; ++r)
                    *reinterpret_cast<float4*>(s_df + frag_row(ty, r) * 8 + tx * 4) = make_float4(a[r][0], a[r][1], a[r][2], a[r][3]);
            }
            __syncthreads();
            if constexpr (STOP) { if (tid < TILE_M && stop_row_live(smem, tid)) volume_scatter<DET, FAST>(sc, io, bw, s_df, si, tid, det, scr); }
            else if (tid < TILE_M && valid) volume_scatter<DET, FAST>(sc, io, bw, s_df, si, tid, det, scr);   // trilinear scatter
        }
        __syncthreads();
    }
    if constexpr (STOP) stop_finish(smem, stop, tid);
}

// ---- per-CTA accumulators -> the 22 tensors in nn.Linear layout ---------------------------------------------
struct GradOut { float* p[MVSN_N_MLP_TENSORS]; };

__global__ void mlp_grad_reduce_kernel(const float* __restrict__ grads, int n_ctas, GradOut out) {
    // blockIdx.y = tensor index; threads enumerate its elements with the output-row index fastest (coalesced reads)
    const int t = blockIdx.y;
    int rows, cols;             // nn.Linear weight [rows][cols] or bias [rows] (cols = 1)
    switch (t) {
        case 0: rows = 128; cols = 63; break;
        case 2: case 4: case 6: case 8: case 16: rows = 128; cols = 128; break;
        case 10: rows = 128; cols = 191; break;
        case 12: rows = 128; cols = 20; break;
        case 14: rows = 64; cols = 131; break;
        case 18: rows = 1; cols = 128; break;
        case 20: rows = 3; cols = 64; break;
        case 15: rows = 64; cols = 1; break;
        case 19: rows = 1; cols = 1; break;
        case 21: rows = 3; cols = 1; break;
        default: rows = 128; cols = 1; break;          // biases 1,3,5,7,9,11,13,17
    }
    const int total = rows * cols;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int n = i % rows, k = i / rows;
        int src;
        switch (t) {
            case 0: src = bwd::G_W0T + k * 128 + n; break;
            case 2: case 4: case 6: case 8: src = bwd::G_W14T + (t / 2 - 1) * 16384 + k * 128 + n; break;
            case 10: src = k < 63 ? bwd::G_W5PET + k * 128 + n : bwd::G_W5HT + (k - 63) * 128 + n; break;
            case 12: src = bwd::G_WBT + k * 128 + n; break;
            case 14: src = k < 128 ? bwd::G_WVFT + k * 64 + n : bwd::G_WVDT + (k - 128) * 64 + n; break;
            case 16: src = bwd::G_WFT + k * 128 + n; break;
            case 18: src = bwd::G_WA + k; break;
            case 20: src = bwd::G_WR + n * 64 + k; break;
            case 1: case 3: case 5: case 7: case 9: case 11: src = bwd::G_B + (t / 2) * 128 + n; break;
            case 13: src = bwd::G_BB + n; break;
            case 15: src = bwd::G_BV + n; break;
            case 17: src = bwd::G_BF + n; break;
            case 19: src = bwd::G_BR + 3; break;
            default: src = bwd::G_BR + n; break;        // 21
        }
        float s = 0.f;
        for (int c = 0; c < n_ctas; ++c) s += grads[(size_t)c * bwd::GRADS + src];
        out.p[t][n * cols + k] = s;
    }
}

struct MlpPtrsB { const float* p[MVSN_N_MLP_TENSORS]; };

__global__ void pack_dgrad_kernel(MlpPtrsB w, float* __restrict__ out) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (int i = tid; i < 64 * 128; i += nt) out[bwd::D_VF + i] = w.p[14][(i >> 7) * 131 + (i & 127)];
    for (int i = tid; i < 128 * 128; i += nt) {
        out[bwd::D_F + i] = w.p[16][i];
        out[bwd::D_5H + i] = w.p[10][(i >> 7) * 191 + 63 + (i & 127)];
        for (int l = 1; l <= 4; ++l) out[bwd::D_14 + (l - 1) * 16384 + i] = w.p[2 * l][i];
    }
    for (int i = tid; i < 128 * 64; i += nt) out[bwd::D_B + i] = (i & 63) < 20 ? w.p[12][(i >> 6) * 20 + (i & 63)] : 0.f;
}

// ============================== grad_mode MVSN_MLP_TC_HALF: dgrad / wgrad on wgmma ==============================
// render_bwd_tc_kernel is render_bwd_kernel with every trunk / feature / views / pts_bias GEMM of the backward moved
// to wgmma with fp16 operands and fp32 accumulation.  Unchanged: the forward recompute (same fp32 tile, same
// ScratchRecord, so rgb / depth / loss are bit-identical), the compositing scan, the element-wise stages, the bias
// gradients (column sums of the fp32 dpre), the volume scatter and the per-CTA private accumulators.
//
// Operands.  Every GEMM operand is an fp16 tile in shared memory in one "core-matrix" layout: a [rows][cols] matrix
// is stored as 8x8 blocks (128 B, one 16-byte row of 8 consecutive columns per matrix row), blocks row-major.  Read
// as K-major (cols = K) it is a wgmma A operand; read as MN-major (rows = K, cols = N, the transposed-B form) it is
// a B operand.  So each matrix is used in the orientation in which it is produced and no shared-memory transpose
// exists:  wgrad  dW^T[k][n] = sum_r x^T[k][r] dpre[r][n]   A = x^T (the transposed record), B = dpre (row-major)
//          dgrad  dx[r][k]   = sum_n dpre[r][n] W[n][k]      A = dpre,                       B = W (nn.Linear layout)
// dpre is converted once per layer and serves as the B of the wgrad and the A of the dgrad.
//
// Scales.  fp16 cannot hold dpre (~1e-6 .. 1e-10 with the 1/(3 N) loss scale) nor activations (up to 1e5) as they
// are.  Each operand tile carries an exact power-of-two scale 2^e, with e chosen so that the tile's max |v| lies in
// [2^14, 2^15); the fp32 epilogue multiplies by 2^-(eA + eB).  Per tile and per layer, not per row: the wgrad sums
// over rows, so a per-row scale on dpre would not factor out.  Conversions saturate at 65504, so no finite input
// gives inf or NaN.  The weights are rounded unscaled (|w| << 65504).
//
// The three GEMMs of width <= 3 (rgb_linear, alpha_linear and the view-direction columns of views_linears.0) are far
// below the wgmma N of 8; they stay FFMA on operands rounded exactly as fp16 would (round_half), so the whole
// backward has one numerics contract: dpre, x and W rounded to an 11-bit significand, fp32 accumulation.
//
// Schedule: 256 threads = 2 warpgroups; warpgroup wg owns output rows [64 wg, 64 wg + 64) (or, for the 64-row
// wgrads, output columns [64 wg, 64 wg + 64)), one m64n64k16 wgmma per 64 columns per K-step, issued back to back
// and retired with one wait.  Tiles live in the regions the fp32 forward tile no longer needs: x16 and d16 in
// sm.mod, the 64-row positional-encoding tile in sm.pe, the layer's fp16 weights in sm.w (cp.async from the
// per-call fp16 image, issued at the start of the layer so the copy overlaps the element-wise stage and the
// conversions).  Activations are converted from the same per-CTA L2 scratch the fp32 backward reads; dgrad results
// return through sm.h (fp32, row-major) to the fragment layout of the shared element-wise code.  wgrad accumulators
// are added straight from the wgmma registers into the private buffers (each element owned by one thread).
namespace bwdtc {
// fp16 dgrad weight image (halves): each B operand [K = n_out][N = k_in] in the core-matrix layout
constexpr int W_VF = 0;                           // views_linears.0.weight[:, :128]   [64][128]
constexpr int W_F  = W_VF + 64 * 128;             // feature_linear.weight             [128][128]
constexpr int W_5H = W_F + 128 * 128;             // pts_linears.5.weight[:, 63:]      [128][128]
constexpr int W_14 = W_5H + 128 * 128;            // pts_linears.1..4.weight           4 x [128][128]
constexpr int W_B  = W_14 + 4 * 128 * 128;        // pts_bias.weight                   [128][64] (k < 20)
constexpr int WIMG = W_B + 128 * 64;
}  // namespace bwdtc

// element (i, j) of a [rows][cols] core-matrix tile, in halves
__host__ __device__ __forceinline__ int core_off(int i, int j, int cols) {
    return ((i >> 3) * (cols >> 3) + (j >> 3)) * 64 + (i & 7) * 8 + (j & 7);
}
// saturating at +-65504 for finite values; NaN stays NaN, so a NaN operand reaches the gradients as it would in fp32
__device__ __forceinline__ __half to_half_sat(float v) {
    return __float2half_rn(v != v ? v : fminf(fmaxf(v, -65504.f), 65504.f));
}
// round to nearest even at an 11-bit significand, exponent unchanged: the value an fp16 operand carries (scaled)
__device__ __forceinline__ float round_half(float x) {
    const unsigned u = __float_as_uint(x);
    return __uint_as_float((u + 0xFFFu + ((u >> 13) & 1u)) & ~0x1FFFu);
}
__device__ __forceinline__ float exp2i(int e) { return __int_as_float((127 + e) << 23); }   // |e| <= 126

__global__ void pack_dgrad_half_kernel(MlpPtrsB w, __half* __restrict__ out) {
    using namespace bwdtc;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (int i = tid; i < 64 * 128; i += nt) {
        const int n = i >> 7, k = i & 127;
        out[W_VF + core_off(n, k, 128)] = to_half_sat(w.p[14][n * 131 + k]);
    }
    for (int i = tid; i < 128 * 128; i += nt) {
        const int n = i >> 7, k = i & 127, o = core_off(n, k, 128);
        out[W_F + o] = to_half_sat(w.p[16][i]);
        out[W_5H + o] = to_half_sat(w.p[10][n * 191 + 63 + k]);
        for (int l = 1; l <= 4; ++l) out[W_14 + (l - 1) * 16384 + o] = to_half_sat(w.p[2 * l][i]);
    }
    for (int i = tid; i < 128 * 64; i += nt) {
        const int n = i >> 6, k = i & 63;
        out[W_B + core_off(n, k, 64)] = to_half_sat(k < 20 ? w.p[12][n * 20 + k] : 0.f);
    }
}

// Block-wide max |v| -> the exponent e of the tile's scale 2^e (max * 2^e in [2^14, 2^15); e = 0 for an all-zero
// tile; clamped to +-62 so that 2^-(eA + eB) is a normal float).  Three rotating slots: use i reads slot i % 3
// after the barrier and clears slot (i + 2) % 3, whose last reader passed the barrier of use i and whose next writer
// comes after the barrier of use i + 1.
__device__ __forceinline__ int block_scale_exp(float m, unsigned* s_amax, int& i, int tid) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) atomicMax(s_amax + i % 3, __float_as_uint(m));
    __syncthreads();
    const unsigned b = s_amax[i % 3];
    if (tid == 0) s_amax[(i + 2) % 3] = 0u;
    ++i;
    if (b == 0u) return 0;
    const int e = 14 - ((int)(b >> 23) - 127);
    return e < -62 ? -62 : (e > 62 ? 62 : e);
}

// fp32 [rows][cols] (row stride ld floats, shared or global) -> scaled fp16 core-matrix tile; returns the exponent.
// Ends with the tile visible to wgmma (proxy fence + barrier).
__device__ __forceinline__ int stage_half(const float* src, int ld, int rows, int cols, __half* dst, unsigned* s_amax,
                                          int& amax_i, int tid) {
    const int upr = cols >> 3, units = rows * upr;
    float m = 0.f;
    for (int u = tid; u < units; u += 256) {
        const float* p = src + (u / upr) * ld + (u % upr) * 8;
        const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
        m = fmaxf(m, fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))),
                           fmaxf(fmaxf(fabsf(b.x), fabsf(b.y)), fmaxf(fabsf(b.z), fabsf(b.w)))));
    }
    const int e = block_scale_exp(m, s_amax, amax_i, tid);
    const float s = exp2i(e);
    for (int u = tid; u < units; u += 256) {
        const int r = u / upr, c8 = u % upr;
        const float* p = src + r * ld + c8 * 8;
        const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
        __half2 h[4] = {__halves2half2(to_half_sat(a.x * s), to_half_sat(a.y * s)), __halves2half2(to_half_sat(a.z * s), to_half_sat(a.w * s)),
                        __halves2half2(to_half_sat(b.x * s), to_half_sat(b.y * s)), __halves2half2(to_half_sat(b.z * s), to_half_sat(b.w * s))};
        *reinterpret_cast<uint4*>(dst + core_off(r, c8 * 8, cols)) = *reinterpret_cast<const uint4*>(h);
    }
    hop::fence_proxy_async();
    __syncthreads();
    return e;
}

// fp16 weight operand (a contiguous slice of the image) -> sm.w by cp.async; completed by load_w_wait
__device__ __forceinline__ void load_w_issue(const __half* src, int halves, __half* dst, int tid) {
    for (int i = tid; i < halves / 8; i += 256) cp_async16(dst + i * 8, src + i * 8);
    cp_async_commit();
}
__device__ __forceinline__ void load_w_wait() {
    cp_async_wait<0>();
    hop::fence_proxy_async();
    __syncthreads();
}

// d[h] = this warpgroup's 64 rows x columns [64 h, 64 h + 64) of A[.][K] * B[K][.]:  a = the warpgroup's first A row
// (core-matrix tile with K columns), b = its first B column (core-matrix tile with ncols columns).
template <int NH, int K>
__device__ __forceinline__ void tc_gemm(float (&d)[NH][32], const __half* a, const __half* b, int ncols) {
    const uint32_t sa = hop::smem_u32(a), sb = hop::smem_u32(b);
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) d[h][i] = 0.f;
    hop::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < K / 16; ++ks) {
        const uint64_t da = hop::desc_nosw(sa + ks * 256, 128, K * 16);
#pragma unroll
        for (int h = 0; h < NH; ++h)
            hop::WgmmaTB<64>::ss(d[h], da, hop::desc_nosw(sb + ks * 32 * ncols + h * 1024, ncols * 16, 128), 1);
    }
    hop::wgmma_commit();
    hop::wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < NH; ++h) hop::reg_fence(d[h]);
}

// accumulator -> row-major fp32 [.][ld] (ACC: += into a private gradient buffer; else: store), times `scale`.
// Element d[h][4 j + 2 hh + e] is row row0 + 16 w + g + 8 hh, column col0 + 64 h + 8 j + 2 q + e.
template <bool ACC, int NH>
__device__ __forceinline__ void tc_write(const float (&d)[NH][32], float scale, float* dst, int ld, int row0, int col0, int tid) {
    const int t = tid & 127, w = t >> 5, g = (t >> 2) & 7, q = t & 3;
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                float2* p = reinterpret_cast<float2*>(dst + (row0 + 16 * w + g + 8 * hh) * ld + col0 + 64 * h + 8 * j + 2 * q);
                float2 v = make_float2(d[h][4 * j + 2 * hh] * scale, d[h][4 * j + 2 * hh + 1] * scale);
                if (ACC) { const float2 o = *p; v.x += o.x; v.y += o.y; }
                *p = v;
            }
}

// row-major fp32 [128][H_LD] (shared) -> the thread's fragment; barriers on both sides, so the caller may overwrite
// the source right after
__device__ __forceinline__ void frag_load_rm(float (&acc)[8][8], const float* src, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const float* p = src + frag_row(ty, r) * H_LD + tx * 4;
        const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 64);
        acc[r][0] = a.x; acc[r][1] = a.y; acc[r][2] = a.z; acc[r][3] = a.w;
        acc[r][4] = b.x; acc[r][5] = b.y; acc[r][6] = b.z; acc[r][7] = b.w;
    }
    __syncthreads();
}

// ============================== grad_mode MVSN_GRAD_TC_FULL: the forward recompute on wgmma too =====================
// tile_mlp_tc replaces tile_mlp in render_bwd_tc_kernel<.., FULL = true> (the rays entries); the backward half of the
// kernel is unchanged.  Arithmetic of the recompute's MLP:
//   * GEMMs with N >= 64 on wgmma, fp16 operands, fp32 accumulation: pts_bias (K 20 -> 32), layer 0 (K 63 -> 64),
//     layers 1-4, layer 5 (encoding 64 + h 128), feature_linear, and the 128 feature columns of views_linears.0.
//   * Front-end operands (encoding, features) unscaled; hidden activations and f carry a power-of-two scale 2^e per
//     sample row, its maximum |v| in [2^14, 2^15) (e = 0 for a zero row, clamped to +-62).  A row's result depends on
//     that row only, so the STOP phase-B recompute repeats phase A bit for bit and a ray's outputs do not depend on the
//     other rays of the batch.  Layer 5's encoding part is accumulated unscaled and the accumulator rows are then
//     multiplied by 2^e (exact) before the h part.  Weights unscaled.  Conversions cvt.rn.satfinite.
//   * The heads of width <= 3 (alpha_linear, rgb_linear, the view-direction columns of views_linears.0): FFMA on
//     operands rounded as fp16 rounds them (round_half), as in the backward.
//   * Biases, modulation product, ReLU, sigmoid, alpha, and everything outside the MLP: fp32.
// Schedule: warpgroup wg owns rows [64 wg, 64 wg + 64); A operands live in registers in the accumulator layout (the
// front-end ones are read from the fp32 rows in sm.pe / sm.h), so a layer's output converts straight into the next
// layer's A.  B operands are the fp16 weight image (the dgrad image read K-major, plus W_0 / W_5P), streamed by
// cp.async through three 32 KB buffers (sm.w and two in sm.mod), two loads ahead.  The tile leaves what tile_mlp
// leaves: sigma / (r, g, b, alpha) per row, hv in sm.mod, and the ScratchRecord of this mode's fp32 values.
namespace bwdtc {
constexpr int W_0  = WIMG;                        // pts_linears.0.weight              [128][64] (k < 63)
constexpr int W_5P = W_0 + 128 * 64;              // pts_linears.5.weight[:, :63]      [128][64] (k < 63)
constexpr int WIMG_FULL = W_5P + 128 * 64;
}  // namespace bwdtc

__global__ void pack_fwd_half_kernel(MlpPtrsB w, __half* __restrict__ out) {
    using namespace bwdtc;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (int i = tid; i < 128 * 64; i += nt) {
        const int n = i >> 6, k = i & 63, o = core_off(n, k, 64);
        out[W_0 + o] = to_half_sat(k < 63 ? w.p[0][n * 63 + k] : 0.f);
        out[W_5P + o] = to_half_sat(k < 63 ? w.p[10][n * 191 + k] : 0.f);
    }
}

// two fp32 -> packed fp16x2 (low half = first argument), saturating
__device__ __forceinline__ uint32_t cvt_h2_satf(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;\n" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
// exponent e of a row's scale 2^e: m * 2^e in [2^14, 2^15) (block_scale_exp's rule, for one row)
__device__ __forceinline__ int row_exp(float m) {
    const unsigned b = __float_as_uint(m);
    if (b == 0u) return 0;
    const int e = 14 - ((int)(b >> 23) - 127);
    return e < -62 ? -62 : (e > 62 ? 62 : e);
}
// accumulator v (v[i]: row a if (i & 2) == 0, else row b) -> the next GEMM's A registers, each row scaled to its own
// exponent (ea / eb out); the four threads of a quad hold a whole row
template <int NV>
__device__ __forceinline__ void to_operand(const float (&v)[NV], uint32_t (&a)[NV / 2], int& ea, int& eb) {
    float ma = 0.f, mb = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i += 4) {
        ma = fmaxf(ma, fmaxf(fabsf(v[i]), fabsf(v[i + 1])));
        mb = fmaxf(mb, fmaxf(fabsf(v[i + 2]), fabsf(v[i + 3])));
    }
    ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 1)); ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 2));
    mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 1)); mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 2));
    ea = row_exp(ma); eb = row_exp(mb);
    const float sa = exp2i(ea), sb = exp2i(eb);
#pragma unroll
    for (int i = 0; i < NV; i += 2) {
        const float s = (i & 2) ? sb : sa;
        a[i >> 1] = cvt_h2_satf(v[i] * s, v[i + 1] * s);
    }
}
// KS K-steps of an unscaled fp32 front-end operand (rows of `src`, stride ld) -> A registers of the warpgroup's rows
template <int KS>
__device__ __forceinline__ void front_operand(uint32_t (&a)[KS * 4], const float* src, int ld, int tid) {
    const int t = tid & 127, w = t >> 5, g = (t >> 2) & 7, q = t & 3, row = 64 * (tid >> 7) + 16 * w + g;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 v = *reinterpret_cast<const float2*>(src + (row + 8 * (i & 1)) * ld + 16 * ks + 8 * (i >> 1) + 2 * q);
            a[ks * 4 + i] = cvt_h2_satf(v.x, v.y);
        }
}
// d (+)= A * W^T for the warpgroup's 64 rows: A from registers (KS K-steps), W [N][ldk] core-matrix tile in shared
// memory read K-major (the B operand of the forward)
template <int N, int KS>
__device__ __forceinline__ void tc_fwd(float (&d)[N / 2], const uint32_t (&a)[KS * 4], const __half* w, int ldk, bool acc) {
    const uint32_t sb = hop::smem_u32(w);
    hop::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
        hop::Wgmma<N>::rs(d, a + 4 * ks, hop::desc_nosw(sb + ks * 256, 128, ldk * 16), (acc || ks > 0) ? 1 : 0);
    hop::wgmma_commit();
    hop::wgmma_wait<0>();
    hop::reg_fence(d);
}
// the record of an N = 128 layer output: dstT[col][row] (128-float rows of the CTA's scratch)
__device__ __forceinline__ void record_T(const float (&v)[64], float* dstT, int tid) {
    const int t = tid & 127, w = t >> 5, g = (t >> 2) & 7, q = t & 3, row = 64 * (tid >> 7) + 16 * w + g;
#pragma unroll
    for (int i = 0; i < 64; ++i) dstT[(8 * (i >> 2) + 2 * q + (i & 1)) * 128 + row + 8 * ((i >> 1) & 1)] = v[i];
}
// cp.async weight loads up to the last N outstanding are complete and visible to wgmma, and every thread is past
// the GEMMs before this barrier
template <int N>
__device__ __forceinline__ void load_w_ready() {
    cp_async_wait<N>();
    hop::fence_proxy_async();
    __syncthreads();
}

// The forward MLP of a tile whose front end is complete (all 256 threads, after the barrier behind the front end).
// Leaves sm.sig, sm.rgb (written by the quad's first thread of each row), hv in sm.mod [128][HV_LD], and the
// ScratchRecord (S_MODT, S_HT, S_FT) in scr; no closing barrier.
__device__ __forceinline__ void tile_mlp_tc(const TileSmem& sm, const float* __restrict__ wts, const __half* __restrict__ wh,
                                            float* scr, int tid) {
    using namespace bwdtc;
    const int t = tid & 127, w = t >> 5, g = (t >> 2) & 7, q = t & 3;
    const int row_a = 64 * (tid >> 7) + 16 * w + g, row_b = row_a + 8;
    __half* const buf0 = reinterpret_cast<__half*>(sm.w);
    __half* const buf1 = reinterpret_cast<__half*>(sm.mod);
    __half* const buf2 = buf1 + 128 * 128;
    auto bias2 = [&](int base, int j) { return __ldg(reinterpret_cast<const float2*>(wts + base + 8 * j + 2 * q)); };
    float acc[64], mod[64];
    uint32_t a[32];
    int ea = 0, eb = 0;
    // the epilogue of a trunk layer: h = relu((acc 2^-e + b) * mod), recorded; then the next A operand
    auto trunk_epilogue = [&](int bias, int l) {
        const float ia = exp2i(-ea), ib = exp2i(-eb);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float2 b = bias2(bias, j);
#pragma unroll
            for (int i = 4 * j; i < 4 * j + 4; ++i)
                acc[i] = fmaxf((acc[i] * ((i & 2) ? ib : ia) + ((i & 1) ? b.y : b.x)) * mod[i], 0.f);
        }
        record_T(acc, scr + bwd::S_HT + l * 16384, tid);
        to_operand(acc, a, ea, eb);
    };

    load_w_issue(wh + W_B, 128 * 64, buf0, tid);                   // the weight stream: load i -> buffer i % 3
    load_w_issue(wh + W_0, 128 * 64, buf1, tid);
    {                                                               // modulation = pts_bias(feat) + bb (K 32)
        uint32_t af[8];
        front_operand<2>(af, sm.h, FEAT_LD, tid);
        load_w_ready<1>();
        load_w_issue(wh + W_14, 128 * 128, buf2, tid);
        tc_fwd<128, 2>(acc, af, buf0, 64, false);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float2 b = bias2(w32::BB, j);
#pragma unroll
            for (int i = 4 * j; i < 4 * j + 4; ++i) mod[i] = acc[i] + ((i & 1) ? b.y : b.x);
        }
        record_T(mod, scr + bwd::S_MODT, tid);
    }
    {                                                               // layer 0: encoding (K 64)
        uint32_t ap[16];
        front_operand<4>(ap, sm.pe, PE_LD, tid);
        load_w_ready<1>();
        load_w_issue(wh + W_14 + 16384, 128 * 128, buf0, tid);
        tc_fwd<128, 4>(acc, ap, buf1, 64, false);
        ea = eb = 0;
        trunk_epilogue(w32::B0, 0);
    }
#pragma unroll 1
    for (int l = 1; l <= 4; ++l) {                                  // layers 1..4: load l + 1 in buffer (l + 1) % 3
        load_w_ready<1>();
        if (l <= 2) load_w_issue(wh + W_14 + (l + 1) * 16384, 128 * 128, l == 1 ? buf1 : buf2, tid);
        else        load_w_issue(wh + (l == 3 ? W_5P : W_5H), l == 3 ? 128 * 64 : 128 * 128, l == 3 ? buf0 : buf1, tid);
        const int nb = (l + 1) % 3;
        tc_fwd<128, 8>(acc, a, nb == 0 ? buf0 : nb == 1 ? buf1 : buf2, 128, false);
        trunk_epilogue(w32::W1 + (l - 1) * w32::LSTR + 128 * 128, l);
    }
    {                                                               // layer 5: [encoding | h] (skip connection)
        uint32_t ap[16];
        front_operand<4>(ap, sm.pe, PE_LD, tid);
        load_w_ready<1>();                                          // load 6: W_5P in buf0
        load_w_issue(wh + W_F, 128 * 128, buf2, tid);
        tc_fwd<128, 4>(acc, ap, buf0, 64, false);
        const float sa = exp2i(ea), sb = exp2i(eb);                 // to the scale of the h rows (exact)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] *= (i & 2) ? sb : sa;
        load_w_ready<1>();                                          // load 7: W_5H in buf1
        load_w_issue(wh + W_VF, 64 * 128, buf0, tid);
        tc_fwd<128, 8>(acc, a, buf1, 128, true);
        trunk_epilogue(w32::B5, 5);
    }
    float sig_a, sig_b;
    {                                                               // sigma = relu(alpha_linear(h6)): FFMA, round_half
        float pa = 0.f, pb = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float2 wa = bias2(w32::WA, j);
            const float w0 = round_half(wa.x), w1 = round_half(wa.y);
            // h6 = the record just written; acc still holds it
            pa = fmaf(round_half(acc[4 * j]), w0, pa); pa = fmaf(round_half(acc[4 * j + 1]), w1, pa);
            pb = fmaf(round_half(acc[4 * j + 2]), w0, pb); pb = fmaf(round_half(acc[4 * j + 3]), w1, pb);
        }
        pa += __shfl_xor_sync(0xffffffffu, pa, 1); pa += __shfl_xor_sync(0xffffffffu, pa, 2);
        pb += __shfl_xor_sync(0xffffffffu, pb, 1); pb += __shfl_xor_sync(0xffffffffu, pb, 2);
        const float ba = __ldg(wts + w32::BA);
        sig_a = fmaxf(pa + ba, 0.f); sig_b = fmaxf(pb + ba, 0.f);
        if (q == 0) { sm.sig[row_a] = sig_a; sm.sig[row_b] = sig_b; }
    }
    {                                                               // f = feature_linear(h6)
        load_w_ready<1>();                                          // load 8: W_F in buf2
        tc_fwd<128, 8>(acc, a, buf2, 128, false);
        const float ia = exp2i(-ea), ib = exp2i(-eb);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float2 b = bias2(w32::BF, j);
#pragma unroll
            for (int i = 4 * j; i < 4 * j + 4; ++i) acc[i] = acc[i] * ((i & 2) ? ib : ia) + ((i & 1) ? b.y : b.x);
        }
        record_T(acc, scr + bwd::S_FT, tid);
        to_operand(acc, a, ea, eb);
    }
    {                                                               // hv = relu(views_linears.0([f, dir])), rgb, alpha
        float hv[32];
        load_w_ready<0>();                                          // load 9: W_VF in buf0; sm.mod is free after this
        tc_fwd<64, 8>(hv, a, buf0, 128, false);
        const float ia = exp2i(-ea), ib = exp2i(-eb);
        float da[3], db[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) { da[c] = round_half(sm.dir[row_a * 4 + c]); db[c] = round_half(sm.dir[row_b * 4 + c]); }
        float ra[3] = {0.f, 0.f, 0.f}, rb[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float2 bv = bias2(w32::BV, j);
            float2 wd[3], wr[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                wd[c] = bias2(w32::WVD + c * 64, j); wd[c].x = round_half(wd[c].x); wd[c].y = round_half(wd[c].y);
                wr[c] = bias2(w32::WR + c * 64, j); wr[c].x = round_half(wr[c].x); wr[c].y = round_half(wr[c].y);
            }
#pragma unroll
            for (int i = 4 * j; i < 4 * j + 4; ++i) {
                const bool hi = i & 1, rb_ = i & 2;
                const float* d = rb_ ? db : da;
                float v = hv[i] * (rb_ ? ib : ia);
                v = fmaf(d[2], hi ? wd[2].y : wd[2].x, fmaf(d[1], hi ? wd[1].y : wd[1].x, fmaf(d[0], hi ? wd[0].y : wd[0].x, v)));
                v = fmaxf(v + (hi ? bv.y : bv.x), 0.f);
                hv[i] = v;
                const float vr = round_half(v);
                float* r = rb_ ? rb : ra;
#pragma unroll
                for (int c = 0; c < 3; ++c) r[c] = fmaf(vr, hi ? wr[c].y : wr[c].x, r[c]);
            }
            const int col = 8 * j + 2 * q;
            *reinterpret_cast<float2*>(sm.mod + row_a * HV_LD + col) = make_float2(hv[4 * j], hv[4 * j + 1]);
            *reinterpret_cast<float2*>(sm.mod + row_b * HV_LD + col) = make_float2(hv[4 * j + 2], hv[4 * j + 3]);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            ra[c] += __shfl_xor_sync(0xffffffffu, ra[c], 1); ra[c] += __shfl_xor_sync(0xffffffffu, ra[c], 2);
            rb[c] += __shfl_xor_sync(0xffffffffu, rb[c], 1); rb[c] += __shfl_xor_sync(0xffffffffu, rb[c], 2);
        }
        if (q == 0) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float br = __ldg(wts + w32::BR + c);
                sm.rgb[row_a * 4 + c] = __fdiv_rn(1.f, 1.f + expf(-(ra[c] + br)));
                sm.rgb[row_b * 4 + c] = __fdiv_rn(1.f, 1.f + expf(-(rb[c] + br)));
            }
            sm.rgb[row_a * 4 + 3] = 1.f - expf(-sig_a);
            sm.rgb[row_b * 4 + 3] = 1.f - expf(-sig_b);
        }
    }
}

template <bool DET, bool FAST, bool STOP = false, bool FULL = false>
__global__ void __launch_bounds__(256, 1)
render_bwd_tc_kernel(const SceneDev sc, const RenderIO io, const BwdIO bw, const float* __restrict__ wts,
                     const __half* __restrict__ wh, const DetIO det, const float* __restrict__ jitter, const StopIO stop) {
    using namespace bwdtc;
    extern __shared__ __align__(16) float smem[];
    const TileSmem sm(smem);
    float* s_T    = sm.tail;
    float* s_g    = s_T + TILE_M;
    float* s_df   = s_g + TILE_M * 4;
    __half* pe16  = reinterpret_cast<__half*>(sm.pe);         // [64][128]  peT: A of the layer-5 / layer-0 pe wgrads
    __half* x16   = reinterpret_cast<__half*>(sm.mod);        // [<=128][128] x^T: A of the wgrads
    __half* d16   = x16 + 128 * 128;                           // [128][<=128] dpre: B of the wgrads, A of the dgrads
    __half* w16   = reinterpret_cast<__half*>(sm.w);          // [<=128][128] W: B of the dgrads
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, wg = tid >> 7;
    __shared__ Cams cams;
    __shared__ unsigned s_amax[3];
    load_cams(sc, &cams, tid);
    if (tid < 3) s_amax[tid] = 0u;
    int amax_i = 0;

    float* scr = bw.scratch + (size_t)blockIdx.x * bwd::SCRATCH;
    float* G = bw.grads + (size_t)blockIdx.x * bwd::GRADS;
    for (int i = tid; i < bwd::GRADS; i += 256) G[i] = 0.f;
    for (int i = tid; i < 32 * 128; i += 256) scr[bwd::S_FEATT + 32 * 128 + i] = 0.f;
    if constexpr (STOP) stop_init(smem, tid);
    __syncthreads();

    const int N = io.N, S = io.S;
    const int R = TILE_M / S;
    const int ngroups = (N + R - 1) / R;

    for (int grp = blockIdx.x; STOP || grp < ngroups; grp += gridDim.x) {
        if constexpr (STOP) { if (!stop_next_tile(smem, stop, grp, ngroups, R, S, N, tid)) break; }
        // =============================== forward recompute (the fp32 tile; FULL: tile_mlp_tc) ==========
        bool valid = false;
        size_t si = 0;
        if (tid < TILE_M) {
            if constexpr (STOP) {
                int ray, s_idx;
                valid = stop_row(smem, tid, ray, s_idx);
                si = (size_t)ray * S + s_idx;
                tile_front_end<FAST>(sc, cams, io, sm, tid, ray, s_idx, valid, ScratchRecord{scr}, jitter);
            } else {
                const int r_in = tid / S, s_idx = tid - r_in * S, ray = grp * R + r_in;
                valid = r_in < R && ray < N;
                si = (size_t)ray * S + s_idx;
                tile_front_end<FAST>(sc, cams, io, sm, tid, ray, s_idx, valid, ScratchRecord{scr}, jitter);
            }
        }
        __syncthreads();
        if constexpr (FULL) tile_mlp_tc(sm, wts, wh, scr, tid);
        else tile_mlp(sm, wts, tid, ScratchRecord{scr});
        __syncthreads();
        composite_scan<DET, STOP>(sc, bw, sm, s_T, s_g, grp, R, S, N, tid, det, &stop, smem);
        if constexpr (STOP) {
            __syncthreads();
            if (stop_defer(smem, stop, grp, ngroups, R, S, N, tid)) continue;
        }
        load_w_issue(wh + W_VF, 64 * 128, w16, tid);
        __syncthreads();
        const int e_pe = stage_half(scr + bwd::S_PET, 128, 64, 128, pe16, s_amax, amax_i, tid);

        // =============================== heads (N <= 3: FFMA on fp16-rounded operands) ================
        if (tid < 64) {
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
            for (int r = 0; r < TILE_M; ++r) {
                const float h = round_half(sm.mod[r * HV_LD + tid]);
                a0 = fmaf(round_half(s_g[r * 4]), h, a0); a1 = fmaf(round_half(s_g[r * 4 + 1]), h, a1);
                a2 = fmaf(round_half(s_g[r * 4 + 2]), h, a2);
            }
            G[bwd::G_WR + tid] += a0; G[bwd::G_WR + 64 + tid] += a1; G[bwd::G_WR + 128 + tid] += a2;
        } else if (tid < 68) {
            const int c = tid - 64;
            float a = 0.f;
            for (int r = 0; r < TILE_M; ++r) a += s_g[r * 4 + c];
            G[bwd::G_BR + c] += a;
        }
        {
            // d hv_pre[r][j] = (hv > 0) * sum_c d rgb_pre[r][c] Wr[c][j]  -> sm.h (fp32, row-major)
            const float4 w0 = __ldg(reinterpret_cast<const float4*>(wts + w32::WR + tx * 4));
            const float4 w1 = __ldg(reinterpret_cast<const float4*>(wts + w32::WR + 64 + tx * 4));
            const float4 w2 = __ldg(reinterpret_cast<const float4*>(wts + w32::WR + 128 + tx * 4));
            const float wr[3][4] = {{round_half(w0.x), round_half(w0.y), round_half(w0.z), round_half(w0.w)},
                                    {round_half(w1.x), round_half(w1.y), round_half(w1.z), round_half(w1.w)},
                                    {round_half(w2.x), round_half(w2.y), round_half(w2.z), round_half(w2.w)}};
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const int row = frag_row(ty, r);
                const float d0 = round_half(s_g[row * 4]), d1 = round_half(s_g[row * 4 + 1]), d2 = round_half(s_g[row * 4 + 2]);
                const float4 hv = *reinterpret_cast<const float4*>(sm.mod + row * HV_LD + tx * 4);
                const float hvv[4] = {hv.x, hv.y, hv.z, hv.w};
                float o[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) o[c] = hvv[c] > 0.f ? fmaf(d2, wr[2][c], fmaf(d1, wr[1][c], d0 * wr[0][c])) : 0.f;
                *reinterpret_cast<float4*>(sm.h + row * H_LD + tx * 4) = make_float4(o[0], o[1], o[2], o[3]);
            }
        }
        __syncthreads();                                        // hv (sm.mod) no longer needed; d hv_pre complete
        if (tid < 64) {                                         // d bv, d Wv[:, 128:131]^T
            float sb = 0.f, s0 = 0.f, s1 = 0.f, s2 = 0.f;
            for (int r = 0; r < TILE_M; ++r) {
                const float d = sm.h[r * H_LD + tid], dr = round_half(d);
                sb += d;
                s0 = fmaf(round_half(sm.dir[r * 4]), dr, s0); s1 = fmaf(round_half(sm.dir[r * 4 + 1]), dr, s1);
                s2 = fmaf(round_half(sm.dir[r * 4 + 2]), dr, s2);
            }
            G[bwd::G_BV + tid] += sb;
            G[bwd::G_WVDT + tid] += s0; G[bwd::G_WVDT + 64 + tid] += s1; G[bwd::G_WVDT + 128 + tid] += s2;
        }
        const int e_dv = stage_half(sm.h, H_LD, 128, 64, d16, s_amax, amax_i, tid);
        const int e_f = stage_half(scr + bwd::S_FT, 128, 128, 128, x16, s_amax, amax_i, tid);
        float d[2][32];
        {
            float d1[1][32];                                    // d Wv_f^T[k][j] = sum_r fT[k][r] d hv_pre[r][j]
            tc_gemm<1, 128>(d1, x16 + wg * 64 * 128, d16, 64);
            tc_write<true>(d1, exp2i(-(e_f + e_dv)), G + bwd::G_WVFT, 64, 64 * wg, 0, tid);
        }
        load_w_wait();                                          // d f[r][k] = sum_j d hv_pre[r][j] Wv[j][k]
        tc_gemm<2, 64>(d, d16 + wg * 64 * 64, w16, 128);
        tc_write<false>(d, exp2i(-e_dv), sm.h, H_LD, 64 * wg, 0, tid);
        __syncthreads();
        load_w_issue(wh + W_F, 128 * 128, w16, tid);
        colsum_accumulate(sm.h, H_LD, 128, G + bwd::G_BF, tid); // d bf
        const int e_df = stage_half(sm.h, H_LD, 128, 128, d16, s_amax, amax_i, tid);
        const int e_h6 = stage_half(scr + bwd::S_HT + 5 * 16384, 128, 128, 128, x16, s_amax, amax_i, tid);
        tc_gemm<2, 128>(d, x16 + wg * 64 * 128, d16, 128);      // d Wf^T[k][n] = sum_r h6T[k][r] d f[r][n]
        tc_write<true>(d, exp2i(-(e_h6 + e_df)), G + bwd::G_WFT, 128, 64 * wg, 0, tid);
        if (tid < TILE_M) {                                     // d wa[k] = sum_r d sigma_pre[r] h6T[k][r]
            const float* h6 = scr + bwd::S_HT + 5 * 16384 + tid * 128;
            float s = 0.f;
            for (int r = 0; r < TILE_M; ++r) s = fmaf(round_half(s_g[r * 4 + 3]), round_half(h6[r]), s);
            G[bwd::G_WA + tid] += s;
        }
        load_w_wait();                                          // d h6 = d f Wf + d sigma_pre (x) wa
        tc_gemm<2, 128>(d, d16 + wg * 64 * 128, w16, 128);
        tc_write<false>(d, exp2i(-e_df), sm.h, H_LD, 64 * wg, 0, tid);
        float acc[8][8];
        frag_load_rm(acc, sm.h, tid);
        {
            const float4 al = __ldg(reinterpret_cast<const float4*>(wts + w32::WA + tx * 4));
            const float4 ah = __ldg(reinterpret_cast<const float4*>(wts + w32::WA + 64 + tx * 4));
            const float wa[8] = {round_half(al.x), round_half(al.y), round_half(al.z), round_half(al.w),
                                 round_half(ah.x), round_half(ah.y), round_half(ah.z), round_half(ah.w)};
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const float ds = round_half(s_g[frag_row(ty, r) * 4 + 3]);
#pragma unroll
                for (int n = 0; n < 8; ++n) acc[r][n] = fmaf(ds, wa[n], acc[r][n]);
            }
        }

        // =============================== trunk, layers 5..0 ==========================================
#pragma unroll 1
        for (int l = 5; l >= 0; --l) {
            trunk_elementwise(acc, scr, l, tid);
            frag_store_rm(acc, sm.h, H_LD, tid);
            if (l >= 1) load_w_issue(wh + (l == 5 ? W_5H : W_14 + (l - 1) * 16384), 128 * 128, w16, tid);
            __syncthreads();
            colsum_accumulate(sm.h, H_LD, 128, G + bwd::G_B + l * 128, tid);                 // d b_l
            const int e_d = stage_half(sm.h, H_LD, 128, 128, d16, s_amax, amax_i, tid);
            if (l >= 1) {                                       // d W_l^T[k][n] = sum_r h_l^T[k][r] d pre[r][n]
                const int e_x = stage_half(scr + bwd::S_HT + (l - 1) * 16384, 128, 128, 128, x16, s_amax, amax_i, tid);
                tc_gemm<2, 128>(d, x16 + wg * 64 * 128, d16, 128);
                tc_write<true>(d, exp2i(-(e_x + e_d)), G + (l == 5 ? bwd::G_W5HT : bwd::G_W14T + (l - 1) * 16384), 128, 64 * wg, 0, tid);
            }
            if (l == 5 || l == 0) {                             // positional-encoding part: 64-row A, column half per warpgroup
                float d1[1][32];
                tc_gemm<1, 128>(d1, pe16, d16 + wg * 512, 128);
                tc_write<true>(d1, exp2i(-(e_pe + e_d)), G + (l == 5 ? bwd::G_W5PET : bwd::G_W0T), 128, 0, 64 * wg, tid);
            }
            if (l >= 1) {                                       // d h_l = d pre W_l (h part)
                load_w_wait();
                tc_gemm<2, 128>(d, d16 + wg * 64 * 128, w16, 128);
                tc_write<false>(d, exp2i(-e_d), sm.h, H_LD, 64 * wg, 0, tid);
                frag_load_rm(acc, sm.h, tid);
            }
        }
        // =============================== modulation branch: pts_bias ==================================
        frag_load_T(acc, scr + bwd::S_DMOD, tid);
        frag_store_rm(acc, sm.h, H_LD, tid);
        if (bw.dvol) load_w_issue(wh + W_B, 128 * 64, w16, tid);
        __syncthreads();
        colsum_accumulate(sm.h, H_LD, 128, G + bwd::G_BB, tid);
        const int e_m = stage_half(sm.h, H_LD, 128, 128, d16, s_amax, amax_i, tid);
        const int e_ft = stage_half(scr + bwd::S_FEATT, 128, 64, 128, x16, s_amax, amax_i, tid);
        {
            float d1[1][32];                                    // d Wb^T[k][n] = sum_r featT[k][r] d mod[r][n]
            tc_gemm<1, 128>(d1, x16, d16 + wg * 512, 128);
            tc_write<true>(d1, exp2i(-(e_ft + e_m)), G + bwd::G_WBT, 128, 0, 64 * wg, tid);
        }
        if (bw.dvol) {
            load_w_wait();                                      // d feat[r][k] = sum_n d mod[r][n] Wb[n][k], k < 8
            float d1[1][32];
            tc_gemm<1, 128>(d1, d16 + wg * 64 * 128, w16, 64);
            const int t = tid & 127, w = t >> 5, g = (t >> 2) & 7, q = t & 3;
            const float sc_m = exp2i(-e_m);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
                *reinterpret_cast<float2*>(s_df + (64 * wg + 16 * w + g + 8 * hh) * 8 + 2 * q) =
                    make_float2(d1[0][2 * hh] * sc_m, d1[0][2 * hh + 1] * sc_m);
            __syncthreads();
            if constexpr (STOP) { if (tid < TILE_M && stop_row_live(smem, tid)) volume_scatter<DET, FAST>(sc, io, bw, s_df, si, tid, det, scr); }
            else if (tid < TILE_M && valid) volume_scatter<DET, FAST>(sc, io, bw, s_df, si, tid, det, scr);
        }
        __syncthreads();
    }
    if constexpr (STOP) stop_finish(smem, stop, tid);
}

// ---- fused Adam (torch.optim.Adam: no weight decay, no amsgrad) ---------------------------------------------
struct AdamScalars { float lr, beta1, beta2, eps, bc1, bc2_sqrt; };

__device__ __forceinline__ float adam_update(float p, float g, float& m, float& v, const AdamScalars& a) {
    m = fmaf(a.beta1, m, (1.f - a.beta1) * g);
    v = fmaf(a.beta2, v, (1.f - a.beta2) * g * g);
    const float denom = __fdiv_rn(sqrtf(v), a.bc2_sqrt) + a.eps;
    return p - __fdiv_rn(a.lr, a.bc1) * __fdiv_rn(m, denom);
}

struct AdamTensors { float* p[MVSN_N_MLP_TENSORS]; const float* g[MVSN_N_MLP_TENSORS]; float* m[MVSN_N_MLP_TENSORS];
                     float* v[MVSN_N_MLP_TENSORS]; int n[MVSN_N_MLP_TENSORS]; int count; };

__global__ void adam_tensors_kernel(AdamTensors t, AdamScalars a) {
    for (int k = blockIdx.y; k < t.count; k += gridDim.y)
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < t.n[k]; i += gridDim.x * blockDim.x) {
            float m = t.m[k][i], v = t.v[k][i];
            t.p[k][i] = adam_update(t.p[k][i], t.g[k][i], m, v, a);
            t.m[k][i] = m; t.v[k][i] = v;
        }
}

// volume: the gradient is channels-last [nvox][8] (the scatter target) and is ZEROED here for the next step; parameter and
// moments here are planar [8][nvox] (a checkpoint-layout nn.Parameter); the channels-last case is adam_volume_cl_kernel
__global__ void adam_volume_planar_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                   long long nvox, AdamScalars a) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox; i += (long long)gridDim.x * blockDim.x) {
        float4* g4 = reinterpret_cast<float4*>(g) + 2 * i;
        const float4 ga = g4[0], gb = g4[1];
        g4[0] = make_float4(0.f, 0.f, 0.f, 0.f); g4[1] = make_float4(0.f, 0.f, 0.f, 0.f);
        const float gg[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const long long j = c * nvox + i;
            float mm = m[j], vv = v[j];
            p[j] = adam_update(p[j], gg[c], mm, vv, a);
            m[j] = mm; v[j] = vv;
        }
    }
}

// channels-last parameter: parameter, moments and gradient share one layout, so the update is purely element-wise --
// one float4 per thread, consecutive lanes on consecutive 16 bytes (fully coalesced streams)
__global__ void adam_volume_cl_kernel(float4* __restrict__ p, float4* __restrict__ g, float4* __restrict__ m, float4* __restrict__ v,
                                      long long n4, AdamScalars a) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 gg = g[i];
        g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 pp = p[i], mm = m[i], vv = v[i];
        pp.x = adam_update(pp.x, gg.x, mm.x, vv.x, a); pp.y = adam_update(pp.y, gg.y, mm.y, vv.y, a);
        pp.z = adam_update(pp.z, gg.z, mm.z, vv.z, a); pp.w = adam_update(pp.w, gg.w, mm.w, vv.w, a);
        p[i] = pp; m[i] = mm; v[i] = vv;
    }
}

// ============================== deterministic volume gradient and loss (DET = true) ==============================
// The float-atomic scatter sums each voxel channel's contributions in whatever order the CTAs reach it.  Here the
// backward kernel records each sample's 8 gradients g (volume_scatter<true>) and the max |g| over them, and the
// scatter happens afterwards in integers, which add associatively:
//   det_scatter_kernel  every contribution g * wgt, formed in fp32 exactly as the atomic path forms it, is scaled by
//                       2^e and rounded to int64 (red.global.add.u64 into a zeroed [D,Hp,Wp,8] accumulator).  A channel
//                       receives at most n = N*S contributions (a sample's 8 corners are distinct voxels), each of
//                       magnitude <= max|g| < 2^(em+1), so e = 61 - ceil(log2 n) - em keeps every partial sum within
//                       2^62.  Contributions below half a quantum 2^-e (~ max|g| * n * 2^-62) round to zero.
//                       A non-finite contribution is added as a float to the fp32 gradient itself, so the entries it
//                       touches become NaN / inf as with the float atomics (and in any order).
//   det_convert_kernel  grad += float(acc) * 2^-e: one correctly rounded conversion, then an exact power-of-two scale.
//   loss_reduce_kernel  the per-ray loss terms in a fixed order (one block, fp64 partial sums) -> += loss_out.
// With max|g| == 0 nothing is scattered or converted (the accumulator stays zero).
__device__ __forceinline__ int det_scale_exp(unsigned amax_bits, long long n) {
    const int em = (int)(amax_bits >> 23) - 127;               // max|g| < 2^(em+1); a subnormal max gives em = -127
    const int k = 64 - __clzll(n - 1);                          // n <= 2^k
    return 61 - k - em;                                         // -106 <= e <= 188 for n <= 2^40: a double scale
}

// FAST (the rays entry): each sample's NDC is marched again from io.rays / io.t_steps / jitter by the function the
// backward kernel's front end used (sample_point), so it has the same bits and needs no per-sample record.
// STOP: the samples j >= live[ray] are dead; their records were never written, so they are skipped.
template <bool FAST, bool STOP = false>
__global__ void det_scatter_kernel(const SceneDev sc, const float* __restrict__ ndc, const float* __restrict__ rec,
                                   const unsigned* __restrict__ amax, long long nsamp,
                                   unsigned long long* __restrict__ acc, float* __restrict__ dvol, const RenderIO io,
                                   const float* __restrict__ jitter, const int* __restrict__ live) {
    const unsigned mb = amax[0];
    if (mb == 0u && amax[1] == 0u) return;                      // all-zero gradients
    __shared__ Cams cams;
    if constexpr (FAST) {
        load_cams(sc, &cams, threadIdx.x);
        __syncthreads();
    }
    const double s = __longlong_as_double((long long)(1023 + det_scale_exp(mb, nsamp)) << 52);
    const int W = sc.Wp, H = sc.Hp, D = sc.D;
    // thread t: sample t >> 6, corner (t >> 3) & 7, channel t & 7 -- a warp adds 4 corners x 64 contiguous bytes
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nsamp * 64; t += (long long)gridDim.x * blockDim.x) {
        const long long si = t >> 6;
        const int c = (int)(t >> 3) & 7, ch = (int)t & 7;
        if constexpr (STOP) {
            const int ray = (int)(si / io.S);
            if (si - (long long)ray * io.S >= __ldg(live + ray)) continue;
        }
        const float g = __ldg(rec + si * 8 + ch);
        if (g == 0.f) continue;
        Trilinear tr;
        if constexpr (FAST) {
            const int ray = (int)(si / io.S), s_idx = (int)(si - (long long)ray * io.S);
            float px, py, pz, dx, dy, dz, nx, ny, nz, z;
            sample_point<true, true>(sc, cams, io, ray, s_idx, (size_t)si, px, py, pz, dx, dy, dz, nx, ny, nz, z, jitter);
            tr = trilinear_corners(sc, nx, ny, nz);
        } else {
            tr = trilinear_corners(sc, __ldg(ndc + si * 3), __ldg(ndc + si * 3 + 1), __ldg(ndc + si * 3 + 2));
        }
        const int x = tr.x0 + (c & 1), y = tr.y0 + ((c >> 1) & 1), z = tr.z0 + (c >> 2);
        if ((unsigned)x >= (unsigned)W || (unsigned)y >= (unsigned)H || (unsigned)z >= (unsigned)D) continue;   // zeros padding
        const float wgt = tr.wx[c & 1] * tr.wy[(c >> 1) & 1] * tr.wz[c >> 2];
        const float p = g * wgt;
        const size_t o = (((size_t)z * H + y) * W + x) * 8 + ch;
        if (!(fabsf(p) <= FLT_MAX)) { atomicAdd(dvol + o, p); continue; }
        const long long q = __double2ll_rn((double)p * s);
        if (q != 0) asm volatile("red.global.add.u64 [%0], %1;" ::"l"(acc + o), "l"(q) : "memory");
    }
}

__global__ void det_convert_kernel(const longlong2* __restrict__ acc, const unsigned* __restrict__ amax, long long nsamp,
                                   float2* __restrict__ dvol, long long n2) {
    const unsigned mb = amax[0];
    if (mb == 0u) return;
    const int e = det_scale_exp(mb, nsamp);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
        const longlong2 a = acc[i];
        if ((a.x | a.y) == 0) continue;                         // untouched (or exactly cancelled): the gradient is as it was
        float2 d = dvol[i];
        if (a.x) d.x += ldexpf(__ll2float_rn(a.x), -e);
        if (a.y) d.y += ldexpf(__ll2float_rn(a.y), -e);
        dvol[i] = d;
    }
}

__global__ void __launch_bounds__(1024) loss_reduce_kernel(const float* __restrict__ terms, int n, float* __restrict__ loss) {
    __shared__ double part[1024];
    double a = 0.0;
    for (int i = threadIdx.x; i < n; i += 1024) a += (double)terms[i];
    part[threadIdx.x] = a;
    __syncthreads();
    for (int w = 512; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss += (float)part[0];
}

static int bwd_grid(int N, int S) {
    const int R = TILE_M / S;
    const int ngroups = (N + R - 1) / R;
    return ngroups < sm_count() ? ngroups : sm_count();
}

// f(std::bool_constant<b0>{}, std::bool_constant<b1>{}, ...) for the runtime flags b0, b1, ...: the kernel variant
// the flags select, with every combination instantiated once
template <bool... B, class F>
static int with_flags(F&& f) { return f(std::bool_constant<B>{}...); }
template <bool... B, class F, class... Flags>
static int with_flags(F&& f, bool b, Flags... rest) {
    return b ? with_flags<B..., true>(f, rest...) : with_flags<B..., false>(f, rest...);
}

// One backward-kernel launch of the variant (grad_mode, DET, FAST, STOP); wh is the fp16 weight image (tensor-core
// modes) or unused.  MVSN_GRAD_TC_FULL exists for FAST only (the entries reject it otherwise).
template <bool DET, bool FAST, bool STOP>
static int launch_bwd_kernel(int grad_mode, int grid, const SceneDev& sc, const RenderIO& io, const BwdIO& bw,
                             const float* wts, const __half* wh, const DetIO& dt, const float* jitter, cudaStream_t stream,
                             const StopIO& stop) {
    static bool attr_set[3][64] = {};
    const int v = grad_mode == MVSN_GRAD_TC_FULL ? 2 : grad_mode == MVSN_MLP_TC_HALF ? 1 : 0;
    const void* kfn = (const void*)render_bwd_kernel<DET, FAST, STOP>;
    if (v == 1) kfn = (const void*)render_bwd_tc_kernel<DET, FAST, STOP>;
    if constexpr (FAST) { if (v == 2) kfn = (const void*)render_bwd_tc_kernel<DET, FAST, STOP, true>; }
    const size_t smem = BWD_SMEM_BYTES + (STOP ? STOP_SMEM_BYTES : 0);
    int dev = 0;
    MVSN_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !attr_set[v][dev]) {
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (dev < 64) attr_set[v][dev] = true;
    }
    if (v == 1) render_bwd_tc_kernel<DET, FAST, STOP><<<grid, 256, smem, stream>>>(sc, io, bw, wts, wh, dt, jitter, stop);
    else if (v == 0) render_bwd_kernel<DET, FAST, STOP><<<grid, 256, smem, stream>>>(sc, io, bw, wts, dt, jitter, stop);
    else if constexpr (FAST) render_bwd_tc_kernel<DET, FAST, STOP, true><<<grid, 256, smem, stream>>>(sc, io, bw, wts, wh, dt, jitter, stop);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

}  // namespace

BwdLayout backward_layout(int N, int S, int D, int Hp, int Wp, int grad_mode, bool det, bool stop) {
    BwdLayout l{};
    const bool frozen = D == 0 && Hp == 0 && Wp == 0;
    if (S <= 0 || S > TILE_M || N <= 0 || (det && !frozen && (D <= 0 || Hp <= 0 || Wp <= 0))) return l;
    // the dgrad weight image behind the per-CTA buffers: fp32, or fp16 for the tensor-core kernel (GRAD_TC_FULL: with
    // the forward's two extra weight operands)
    size_t wimg;
    if (grad_mode == MVSN_MLP_FP32) wimg = bwd::DGRAD * sizeof(float);
    else if (grad_mode == MVSN_MLP_TC_HALF) wimg = bwdtc::WIMG * sizeof(__half);
    else if (grad_mode == MVSN_GRAD_TC_FULL) wimg = bwdtc::WIMG_FULL * sizeof(__half);
    else return l;
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t ctas = (size_t)sm_count();              // sized for the widest launch on this device
    size_t end = ctas * (bwd::SCRATCH + bwd::GRADS) * sizeof(float) + wimg;
    // deterministic: (256-byte aligned) the [N] loss terms, and with a volume gradient the two amax words (in a 256-byte
    // slot), the int64 accumulator [D,Hp,Wp,8] right behind them (one memset zeroes both) and the [N*S][8] record
    if (det) {
        const size_t nvox = (size_t)D * Hp * Wp;
        l.loss = up(end);
        l.amax = up(l.loss + (size_t)N * sizeof(float));
        l.acc = l.amax + 256;
        l.rec = up(l.acc + nvox * 8 * sizeof(long long));
        end = nvox ? l.rec + (size_t)N * S * 8 * sizeof(float) : l.amax;
    }
    // early ray termination: (256-byte aligned) the [N] live counts and the CTAs' deferred-ray lists, list_cap (ray, live
    // samples) pairs per CTA: every ray of its phase-A groups
    if (stop) {
        const int R = TILE_M / S, ngroups = (N + R - 1) / R, grid = bwd_grid(N, S);
        l.list_cap = (ngroups + grid - 1) / grid * R;
        l.live = up(end);
        l.list = up(l.live + (size_t)N * sizeof(int));
        end = l.list + (size_t)grid * l.list_cap * sizeof(int2);
    }
    l.total = end;
    return l;
}

int launch_render_backward(const SceneDev& sc, const RenderIO& io, const float* wts_fp32, const BwdCall& call,
                           cudaStream_t stream) {
    const bool fast = io.rays != nullptr, tc = call.grad_mode != MVSN_MLP_FP32, vol = call.dvol != nullptr;
    const BwdLayout l = backward_layout(io.N, io.S, vol ? sc.D : 0, vol ? sc.Hp : 0, vol ? sc.Wp : 0, call.grad_mode,
                                        call.det, call.stop != nullptr);
    MVSN_REQUIRE(call.workspace && call.workspace_bytes >= l.total, MVSN_EWORKSPACE, "%s: workspace %zu < %zu bytes",
                 call.what, call.workspace_bytes, l.total);
    MVSN_REQUIRE(aligned16(call.workspace), MVSN_EALIGN, "%s: workspace must be 16-byte aligned", call.what);
    char* w8 = static_cast<char*>(call.workspace);
    DetIO dt{};
    if (call.det) {
        dt.loss_terms = reinterpret_cast<float*>(w8 + l.loss);
        if (vol) {
            dt.amax = reinterpret_cast<unsigned*>(w8 + l.amax);
            dt.rec = reinterpret_cast<float*>(w8 + l.rec);
            // the workspace is shared between modes and callers may hand it over uninitialised: zero every call
            MVSN_CUDA_CHECK(cudaMemsetAsync(w8 + l.amax, 0, l.rec - l.amax, stream));
        }
    }
    const int grid = bwd_grid(io.N, io.S);
    float* ws = static_cast<float*>(call.workspace);
    const size_t ctas = (size_t)sm_count();
    const mvsn_render_grads& g = *call.g;
    BwdIO bw{};
    bw.g_rgb = g.rgb; bw.target = g.target_rgb; bw.inv_count = g.loss_scale; bw.g_depth = g.depth; bw.g_weights = g.weights;
    bw.g_alpha = g.alpha; bw.g_feat = g.input_feat; bw.dvol = call.dvol; bw.rgb_out = g.rgb_out; bw.depth_out = g.depth_out;
    bw.loss = g.loss_out;
    bw.scratch = ws; bw.grads = ws + ctas * bwd::SCRATCH;
    float* wimg = ws + ctas * (bwd::SCRATCH + bwd::GRADS);   // the dgrad weight image: fp32, or fp16 for the tc kernel
    MlpPtrsB wp;
    for (int i = 0; i < MVSN_N_MLP_TENSORS; ++i) wp.p[i] = call.mlp_w[i];
    __half* wh = reinterpret_cast<__half*>(wimg);
    if (tc) {
        pack_dgrad_half_kernel<<<64, 256, 0, stream>>>(wp, wh);
        if (call.grad_mode == MVSN_GRAD_TC_FULL) {
            MVSN_CUDA_CHECK(cudaGetLastError());
            pack_fwd_half_kernel<<<32, 256, 0, stream>>>(wp, wh);
        }
    } else {
        bw.wd = wimg;
        pack_dgrad_kernel<<<64, 256, 0, stream>>>(wp, wimg);
    }
    MVSN_CUDA_CHECK(cudaGetLastError());
    StopIO st{};
    if (call.stop) {
        st.t_stop = call.stop->t_stop;
        st.live = call.stop->live_samples ? call.stop->live_samples : reinterpret_cast<int*>(w8 + l.live);
        st.list = reinterpret_cast<int2*>(w8 + l.list);
        st.list_cap = l.list_cap;
        st.tiles_done = call.stop->tiles_done;
    }
    const int rc = with_flags([&](auto STOP, auto DET, auto FAST) {
        return launch_bwd_kernel<DET, FAST, STOP>(call.grad_mode, grid, sc, io, bw, wts_fp32, wh, dt, call.jitter, stream, st);
    }, call.stop != nullptr, call.det, fast);
    if (rc) return rc;
    GradOut go;
    for (int i = 0; i < MVSN_N_MLP_TENSORS; ++i) go.p[i] = call.grad_mlp[i];
    mlp_grad_reduce_kernel<<<dim3(16, MVSN_N_MLP_TENSORS), 256, 0, stream>>>(bw.grads, grid, go);
    MVSN_CUDA_CHECK(cudaGetLastError());
    if (call.det && vol) {
        const long long nsamp = (long long)io.N * io.S;
        auto* acc = reinterpret_cast<unsigned long long*>(w8 + l.acc);
        const int gs = cdiv(nsamp * 64, 256) < sm_count() * 16 ? cdiv(nsamp * 64, 256) : sm_count() * 16;
        // io.ndc is NULL for the rays entries, call.jitter and st.live for the entries without them
        with_flags([&](auto STOP, auto FAST) {
            det_scatter_kernel<FAST, STOP><<<gs, 256, 0, stream>>>(sc, io.ndc, dt.rec, dt.amax, nsamp, acc, call.dvol, io,
                                                                   call.jitter, st.live);
            return 0;
        }, call.stop != nullptr, fast);
        MVSN_CUDA_CHECK(cudaGetLastError());
        const long long n2 = (long long)sc.D * sc.Hp * sc.Wp * 4;   // (int64 pair, float pair) per thread step
        const int gc = cdiv(n2, 256) < sm_count() * 8 ? cdiv(n2, 256) : sm_count() * 8;
        det_convert_kernel<<<gc, 256, 0, stream>>>(reinterpret_cast<const longlong2*>(acc), dt.amax, nsamp,
                                                   reinterpret_cast<float2*>(call.dvol), n2);
        MVSN_CUDA_CHECK(cudaGetLastError());
    }
    if (call.det && g.loss_out && g.target_rgb) {               // the terms exist only with the fused loss
        loss_reduce_kernel<<<1, 1024, 0, stream>>>(dt.loss_terms, io.N, g.loss_out);
        MVSN_CUDA_CHECK(cudaGetLastError());
    }
    return MVSN_OK;
}

int launch_adam_tensors(float* const* p, const float* const* g, float* const* m, float* const* v, const int* n, int count,
                        float lr, float beta1, float beta2, float eps, int step, cudaStream_t stream) {
    MVSN_REQUIRE(count >= 0 && count <= MVSN_N_MLP_TENSORS, MVSN_EBADSHAPE, "adam: %d tensors (max %d per call)", count, MVSN_N_MLP_TENSORS);
    if (count == 0) return MVSN_OK;
    AdamTensors t{};
    for (int i = 0; i < count; ++i) { t.p[i] = p[i]; t.g[i] = g[i]; t.m[i] = m[i]; t.v[i] = v[i]; t.n[i] = n[i]; }
    t.count = count;
    const AdamScalars a{lr, beta1, beta2, eps, (float)(1.0 - pow((double)beta1, step)), (float)sqrt(1.0 - pow((double)beta2, step))};
    adam_tensors_kernel<<<dim3(16, count), 256, 0, stream>>>(t, a);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

int launch_adam_volume(float* p, float* g_dhwc, float* m, float* v, long long nvox, int planar, float lr, float beta1,
                       float beta2, float eps, int step, cudaStream_t stream) {
    const AdamScalars a{lr, beta1, beta2, eps, (float)(1.0 - pow((double)beta1, step)), (float)sqrt(1.0 - pow((double)beta2, step))};
    const int grid = sm_count() * 8;
    if (planar) adam_volume_planar_kernel<<<grid, 256, 0, stream>>>(p, g_dhwc, m, v, nvox, a);
    else        adam_volume_cl_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<float4*>(p), reinterpret_cast<float4*>(g_dhwc),
                                                                reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v), 2 * nvox, a);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

}  // namespace mvsn
