// The fp32 FFMA forward tile, written once for the forward render kernel (render_fp32.cu) and the forward recompute
// of the fine-tuning backward kernel (render_bwd.cu), so that the backward differentiates the function the forward
// renders.  A tile is 128 samples, one shared-memory row each:
//   tile_front_end  one row: ray march, NDC, 8-ch trilinear volume fetch, 3-view colour fetch, positional encoding
//   tile_mlp        the MLP (models.py:194-222) over the tile: GEMM passes with 8x8 register blocking whose B operand
//                   is streamed global -> shared with cp.async double buffering, bias / modulation / activation fused
//                   into each pass epilogue; leaves sigma and (r, g, b, alpha) per row
// Both take a recorder, a compile-time hook for what the backward keeps of the forward (NoRecord: nothing).
#pragma once
#include "render_frontend.cuh"

namespace mvsn {

constexpr int TILE_M = 128;
constexpr int PE_LD  = 68;    // 63 PE channels + 1 zero + 4 pad (row stride = 16 banks mod 32)
constexpr int H_LD   = 132;
constexpr int FEAT_LD = 36;   // 20 features + 12 zeros + 4 pad
constexpr int HV_LD  = 68;
constexpr int KCHUNK = 32;


__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// acc[MR][NC/16] += A[16 MR][K] (smem, row stride lda) * Wt[K][NC] (global, streamed through sW).
// Thread (ty, tx) = (tid/16, tid%16) owns rows {4ty..4ty+3, 64+4ty..} (MR = 8; MR = 4: the first four only, i.e. a
// 64-row A) and columns {4tx..4tx+3, NC/2+4tx..} (NC=128) or {4tx..4tx+3} (NC=64).
template <int NC, int MR>
__device__ __forceinline__ void gemm_pass(float (&acc)[MR][NC / 16], const float* sA, int lda, int K,
                                          const float* __restrict__ gW, float* sW, int tid) {
    static_assert(MR == 8 || MR == 4, "8 (128-row A) or 4 (64-row A) rows per thread");
    constexpr int NT = NC / 16;
    constexpr int V4_PER_CHUNK = KCHUNK * NC / 4;
    const int ty = tid >> 4, tx = tid & 15;
    const int nchunks = K / KCHUNK;
    auto issue = [&](int c) {
        const float4* src = reinterpret_cast<const float4*>(gW + (size_t)c * KCHUNK * NC);
        float4* dst = reinterpret_cast<float4*>(sW + (c & 1) * KCHUNK * NC);
        for (int i = tid; i < V4_PER_CHUNK; i += 256) cp_async16(dst + i, src + i);
        cp_async_commit();
    };
    issue(0);
    for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) { issue(c + 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
        __syncthreads();
        const float* w = sW + (c & 1) * KCHUNK * NC;
        const float* a0 = sA + (ty * 4) * lda + c * KCHUNK;
        const float* a1 = sA + (64 + ty * 4) * lda + c * KCHUNK;
#pragma unroll 2
        for (int kk = 0; kk < KCHUNK; kk += 4) {
            float4 av[MR];
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                av[r] = *reinterpret_cast<const float4*>(a0 + r * lda + kk);
                if constexpr (MR == 8) av[4 + r] = *reinterpret_cast<const float4*>(a1 + r * lda + kk);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float b[NT];
                float4 b0 = *reinterpret_cast<const float4*>(w + (kk + j) * NC + tx * 4);
                b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
                if constexpr (NT == 8) {
                    float4 b1 = *reinterpret_cast<const float4*>(w + (kk + j) * NC + NC / 2 + tx * 4);
                    b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
                }
#pragma unroll
                for (int r = 0; r < MR; ++r) {
                    float a = j == 0 ? av[r].x : j == 1 ? av[r].y : j == 2 ? av[r].z : av[r].w;
#pragma unroll
                    for (int n = 0; n < NT; ++n) acc[r][n] = fmaf(a, b[n], acc[r][n]);
                }
            }
        }
        __syncthreads();   // everyone is done with this weight buffer (and, on the last chunk, with sA)
    }
}

template <int MR, int NT> __device__ __forceinline__ void zero_acc(float (&acc)[MR][NT]) {
#pragma unroll
    for (int r = 0; r < MR; ++r)
#pragma unroll
        for (int n = 0; n < NT; ++n) acc[r][n] = 0.f;
}

// Shared-memory prefix of both tile kernels; each kernel's own per-row scalars follow at `tail`.
constexpr int TILE_SMEM_FLOATS = TILE_M * PE_LD + 2 * TILE_M * H_LD + 2 * KCHUNK * 128 + TILE_M * 10;
struct TileSmem {
    float* pe;     // [128][PE_LD] positional encoding
    float* h;      // [128][H_LD]  feature rows ([128][FEAT_LD]), then the hidden layers, then feature_linear
    float* mod;    // [128][H_LD]  modulation, then hv [128][HV_LD]
    float* w;      // 2 x [32][128] streamed weight chunks
    float* dir;    // [128][4] view direction of the row's ray
    float* z;      // [128]
    float* sig;    // [128] sigma = relu(alpha_linear(h))
    float* rgb;    // [128][4] r, g, b, alpha
    float* tail;
    __device__ __forceinline__ explicit TileSmem(float* smem)
        : pe(smem), h(pe + TILE_M * PE_LD), mod(h + TILE_M * H_LD), w(mod + TILE_M * H_LD), dir(w + 2 * KCHUNK * 128),
          z(dir + TILE_M * 4), sig(z + TILE_M), rgb(sig + TILE_M), tail(rgb + TILE_M * 4) {}
};

// Recorder interface.  pe / feat: row `row` of the front end stores column k of its positional-encoding / feature
// row; mod / hidden / feature: every thread, with its fragment of a layer output after the epilogue (hidden l = 0..5
// is h_{l+1}).  The forward records nothing.
struct NoRecord {
    __device__ __forceinline__ void pe(int, int, float) const {}
    __device__ __forceinline__ void feat(int, int, float) const {}
    __device__ __forceinline__ void mod(const float (&)[8][8], int) const {}
    __device__ __forceinline__ void hidden(int, const float (&)[8][8], int) const {}
    __device__ __forceinline__ void feature(const float (&)[8][8], int) const {}
};

// Fragment of thread (ty, tx) = (tid/16, tid%16) in an N=128 pass: rows {4ty+i, 64+4ty+i}, cols {4tx+j, 64+4tx+j}.
__device__ __forceinline__ int frag_row(int ty, int r) { return (r < 4 ? 0 : 64) + ty * 4 + (r & 3); }
__device__ __forceinline__ int frag_col(int tx, int n) { return (n < 4 ? 0 : 64) + tx * 4 + (n & 3); }

// row-major [128][ld] store (shared or global)
__device__ __forceinline__ void frag_store_rm(const float (&acc)[8][8], float* dst, int ld, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        float* p = dst + frag_row(ty, r) * ld + tx * 4;
        *reinterpret_cast<float4*>(p) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
        *reinterpret_cast<float4*>(p + 64) = make_float4(acc[r][4], acc[r][5], acc[r][6], acc[r][7]);
    }
}
// bias add (MODE 0) or relu((acc + bias) * mod) (MODE 1) in place; mod read from shared [128][H_LD]
template <int MODE>
__device__ __forceinline__ void epilogue128(float (&acc)[8][8], const float* __restrict__ bias, const float* s_mod, int tid) {
    const int ty = tid >> 4, tx = tid & 15;
    const float4 bl = __ldg(reinterpret_cast<const float4*>(bias + tx * 4));
    const float4 bh = __ldg(reinterpret_cast<const float4*>(bias + 64 + tx * 4));
    const float b[8] = {bl.x, bl.y, bl.z, bl.w, bh.x, bh.y, bh.z, bh.w};
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int row = frag_row(ty, r);
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            float v = acc[r][n] + b[n];
            if (MODE == 1) v = fmaxf(v * s_mod[row * H_LD + frag_col(tx, n)], 0.f);
            acc[r][n] = v;
        }
    }
}

// Front end of row `row` (threads 0..127): sample s_idx of ray `ray`, as the caller maps rows to samples.  Fills the
// row of sm.pe, the FEAT_LD feature row at the start of sm.h, sm.dir and sm.z; an invalid row gets zeros (and
// cos(0) = 1 in its positional encoding).  With io.input_feat set, the 20 feature channels also go to HBM.
// `jitter`: stratified depths for the FAST march (see sample_point).  VT: the volume storage (see sample_volume).
template <bool FAST, class Rec, typename VT = float>
__device__ __forceinline__ void tile_front_end(const SceneDev& sc, const Cams& cams, const RenderIO& io, const TileSmem& sm,
                                               int row, int ray, int s_idx, bool valid, const Rec& rec,
                                               const float* jitter = nullptr) {
    float pe[3] = {0.f, 0.f, 0.f}, feat[20], dir[3] = {0.f, 0.f, 0.f}, zv = 0.f;
#pragma unroll
    for (int i = 0; i < 20; ++i) feat[i] = 0.f;
    if (valid) {
        const size_t si = (size_t)ray * io.S + s_idx;
        float px, py, pz, dx, dy, dz;
        sample_point<FAST, true>(sc, cams, io, ray, s_idx, si, px, py, pz, dx, dy, dz, pe[0], pe[1], pe[2], zv, jitter);
        view_dir(cams, dx, dy, dz, dir);
        sample_volume<VT>(sc, pe[0], pe[1], pe[2], feat);
#pragma unroll
        for (int v = 0; v < 3; ++v) sample_color(sc, cams, v, px, py, pz, feat + 8 + 4 * v);
        if (io.input_feat) {
            float4* o = reinterpret_cast<float4*>(io.input_feat + si * 20);
#pragma unroll
            for (int i = 0; i < 5; ++i) o[i] = make_float4(feat[4 * i], feat[4 * i + 1], feat[4 * i + 2], feat[4 * i + 3]);
        }
    }
    // positional encoding (models.py:47-51): [x, sin(2^k x) k-major, cos(2^k x) k-major, 0]
    float* pr = sm.pe + row * PE_LD;
    pr[0] = pe[0]; pr[1] = pe[1]; pr[2] = pe[2];
    rec.pe(row, 0, pe[0]); rec.pe(row, 1, pe[1]); rec.pe(row, 2, pe[2]);
    float f = 1.f;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float sn, cs;
            sincosf(pe[j] * f, &sn, &cs);
            pr[3 + 3 * k + j] = sn; pr[33 + 3 * k + j] = cs;
            rec.pe(row, 3 + 3 * k + j, sn); rec.pe(row, 33 + 3 * k + j, cs);
        }
        f *= 2.f;
    }
    pr[63] = 0.f; rec.pe(row, 63, 0.f);
    float* fr = sm.h + row * FEAT_LD;
#pragma unroll
    for (int i = 0; i < 32; ++i) { const float v = i < 20 ? feat[i] : 0.f; fr[i] = v; rec.feat(row, i, v); }
    sm.dir[row * 4 + 0] = dir[0]; sm.dir[row * 4 + 1] = dir[1]; sm.dir[row * 4 + 2] = dir[2];
    sm.z[row] = zv;
}

// The MLP over a tile whose front end is complete (all 256 threads; starts with the tile in shared memory and the
// barrier behind it).  Leaves sigma in sm.sig and (r, g, b, alpha) in sm.rgb, each row written by its own thread
// (tid < 128) with no closing barrier.
template <class Rec>
__device__ __forceinline__ void tile_mlp(const TileSmem& sm, const float* __restrict__ wts, int tid, const Rec& rec) {
    const int ty = tid >> 4, tx = tid & 15;
    {
        float acc[8][8];
        zero_acc(acc);                                                     // modulation = pts_bias(feat)
        gemm_pass<128>(acc, sm.h, FEAT_LD, 32, wts + w32::WB, sm.w, tid);
        epilogue128<0>(acc, wts + w32::BB, nullptr, tid);
        frag_store_rm(acc, sm.mod, H_LD, tid);
        rec.mod(acc, tid);
        __syncthreads();
        zero_acc(acc);                                                     // layer 0: 63 -> 128
        gemm_pass<128>(acc, sm.pe, PE_LD, 64, wts + w32::W0, sm.w, tid);
        epilogue128<1>(acc, wts + w32::B0, sm.mod, tid);
        frag_store_rm(acc, sm.h, H_LD, tid);
        rec.hidden(0, acc, tid);
        __syncthreads();
        for (int l = 0; l < 4; ++l) {                                      // layers 1..4: 128 -> 128
            zero_acc(acc);
            gemm_pass<128>(acc, sm.h, H_LD, 128, wts + w32::W1 + l * w32::LSTR, sm.w, tid);
            epilogue128<1>(acc, wts + w32::W1 + l * w32::LSTR + 128 * 128, sm.mod, tid);
            frag_store_rm(acc, sm.h, H_LD, tid);
            rec.hidden(l + 1, acc, tid);
            __syncthreads();
        }
        zero_acc(acc);                                                     // layer 5: [pe63, h128] -> 128 (skip, models.py:204-205)
        gemm_pass<128>(acc, sm.pe, PE_LD, 64, wts + w32::W5, sm.w, tid);
        gemm_pass<128>(acc, sm.h, H_LD, 128, wts + w32::W5 + 64 * 128, sm.w, tid);
        epilogue128<1>(acc, wts + w32::B5, sm.mod, tid);
        frag_store_rm(acc, sm.h, H_LD, tid);
        rec.hidden(5, acc, tid);
        __syncthreads();
        if (tid < TILE_M) {                                                // sigma = relu(alpha_linear(h6))
            const float4* hr = reinterpret_cast<const float4*>(sm.h + tid * H_LD);
            const float4* wa = reinterpret_cast<const float4*>(wts + w32::WA);
            float s = 0.f;
#pragma unroll 8
            for (int i = 0; i < 32; ++i) {
                const float4 a = hr[i], b = __ldg(wa + i);
                s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); s = fmaf(a.w, b.w, s);
            }
            sm.sig[tid] = fmaxf(s + __ldg(wts + w32::BA), 0.f);
        }
        zero_acc(acc);                                                     // f = feature_linear(h6), in place
        gemm_pass<128>(acc, sm.h, H_LD, 128, wts + w32::WF, sm.w, tid);
        epilogue128<0>(acc, wts + w32::BF, nullptr, tid);
        frag_store_rm(acc, sm.h, H_LD, tid);
        rec.feature(acc, tid);
        __syncthreads();
    }
    {
        float acc[8][4];                                                   // hv = relu(views_linear([f, dir])) : 131 -> 64
        zero_acc(acc);
        gemm_pass<64>(acc, sm.h, H_LD, 128, wts + w32::WV, sm.w, tid);
        const float4 bv = __ldg(reinterpret_cast<const float4*>(wts + w32::BV + tx * 4));
        const float4 wd0 = __ldg(reinterpret_cast<const float4*>(wts + w32::WVD + 0 * 64 + tx * 4));
        const float4 wd1 = __ldg(reinterpret_cast<const float4*>(wts + w32::WVD + 1 * 64 + tx * 4));
        const float4 wd2 = __ldg(reinterpret_cast<const float4*>(wts + w32::WVD + 2 * 64 + tx * 4));
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const int row = frag_row(ty, r);
            const float d0 = sm.dir[row * 4], d1 = sm.dir[row * 4 + 1], d2 = sm.dir[row * 4 + 2];
            float4 o;
            o.x = fmaxf(fmaf(d2, wd2.x, fmaf(d1, wd1.x, fmaf(d0, wd0.x, acc[r][0]))) + bv.x, 0.f);
            o.y = fmaxf(fmaf(d2, wd2.y, fmaf(d1, wd1.y, fmaf(d0, wd0.y, acc[r][1]))) + bv.y, 0.f);
            o.z = fmaxf(fmaf(d2, wd2.z, fmaf(d1, wd1.z, fmaf(d0, wd0.z, acc[r][2]))) + bv.z, 0.f);
            o.w = fmaxf(fmaf(d2, wd2.w, fmaf(d1, wd1.w, fmaf(d0, wd0.w, acc[r][3]))) + bv.w, 0.f);
            *reinterpret_cast<float4*>(sm.mod + row * HV_LD + tx * 4) = o;
        }
        __syncthreads();
    }
    if (tid < TILE_M) {                                                    // rgb = sigmoid(rgb_linear(hv)) ; alpha = 1 - exp(-sigma)
        const float4* hr = reinterpret_cast<const float4*>(sm.mod + tid * HV_LD);   // (renderer.py:18-26)
        float o[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float4* wr = reinterpret_cast<const float4*>(wts + w32::WR + c * 64);
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float4 a = hr[i], b = __ldg(wr + i);
                s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); s = fmaf(a.w, b.w, s);
            }
            s += __ldg(wts + w32::BR + c);
            o[c] = __fdiv_rn(1.f, 1.f + expf(-s));
        }
        sm.rgb[tid * 4 + 0] = o[0]; sm.rgb[tid * 4 + 1] = o[1]; sm.rgb[tid * 4 + 2] = o[2];
        sm.rgb[tid * 4 + 3] = 1.f - expf(-sm.sig[tid]);
    }
}

}  // namespace mvsn
