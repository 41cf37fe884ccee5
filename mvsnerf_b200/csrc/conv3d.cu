// K-B: CostRegNet (models.py:725-769) -- ten bias-free 3x3x3 (transposed) convolutions, each
// followed by InPlaceABN in TRAIN mode (batch statistics, |gamma|+eps, leaky-ReLU 0.01).
//
// Train-mode BN makes every layer end in a grid-wide per-channel reduction, so a layer is one
// kernel that (a) applies the PREVIOUS layer's normalisation + activation while loading its input
// ("normalise on load": activations are stored raw, exactly once), (b) convolves, (c) stores the
// raw result and (d) accumulates per-channel sum / sum of squares (fp32 per CTA, fp64 across CTAs)
// for the NEXT layer's load.  No separate BN or activation pass over any tensor exists, and the
// U-Net skip additions are folded into the consumer's load as a second (tensor, statistics) pair.
//
// Thread mapping: a thread owns a strip of 4 consecutive output voxels along x for CT output
// channels; a warp owns 32 consecutive strips, so input rows are fetched with one 16-byte load per
// lane and the +-1 halo comes from the neighbouring lanes by shuffle.  Weights for the CTA's CT
// output channels sit in shared memory ([cin][27][CT], read as broadcast LDS.128).
#include <cuda_fp16.h>
#include "conv_common.cuh"

namespace mvsn {


// write 4 x CT raw outputs + accumulate batch statistics
template <int CT>
__device__ __forceinline__ void store_and_stats(const ConvArgs& a, float (&acc)[4][CT], bool active, int z, int y,
                                                int x0, int cg, float* s_stat, int tid) {
    const int lane = tid & 31;
    const size_t plane = (size_t)a.Hout * a.Wout, vol = plane * a.Dout;
    const bool vec = (a.Wout & 3) == 0;
#pragma unroll
    for (int c = 0; c < CT; ++c) {
        float s = 0.f, q = 0.f;
        if (active) {
            float* o = a.out + (size_t)(cg * CT + c) * vol + (size_t)z * plane + (size_t)y * a.Wout + x0;
            if (vec) {
                *reinterpret_cast<float4*>(o) = make_float4(acc[0][c], acc[1][c], acc[2][c], acc[3][c]);
#pragma unroll
                for (int i = 0; i < 4; ++i) { s += acc[i][c]; q = fmaf(acc[i][c], acc[i][c], q); }
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (x0 + i < a.Wout) { o[i] = acc[i][c]; s += acc[i][c]; q = fmaf(acc[i][c], acc[i][c], q); }
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, off);
            q += __shfl_xor_sync(0xffffffffu, q, off);
        }
        if (lane == 0) { s_stat[(tid >> 5) * 2 * CT + 2 * c] = s; s_stat[(tid >> 5) * 2 * CT + 2 * c + 1] = q; }
    }
    __syncthreads();
    if (tid < 2 * CT)       // four warp partials -> fixed point -> ONE integer atomic per CTA and slot (order-independent)
        atomicAdd(reinterpret_cast<unsigned long long*>(a.stats_out) + 2 * (cg * CT) + tid,
                  stat_fx(s_stat[tid]) + stat_fx(s_stat[2 * CT + tid]) + stat_fx(s_stat[4 * CT + tid]) + stat_fx(s_stat[6 * CT + tid]));
}

// ------------------------------------------------------------------------------------------
// Conv3d k3 p1, stride 1 or 2
// ------------------------------------------------------------------------------------------
// (Conv3d layers never take a skip sum -- only the transposed ones do -- so in1 is not read here.)
template <int CT, int STRIDE, bool IDENT>
__global__ void __launch_bounds__(128)
conv3d_k3_kernel(const ConvArgs a) {
    extern __shared__ __align__(16) float s_w[];            // [Cin][27][CT]
    __shared__ float s_sc[kMaxCin], s_sh[kMaxCin];
    __shared__ float s_stat[4 * 2 * CT];            // per-warp partial sums (4 warps), combined in fixed point
    const int tid = threadIdx.x, lane = tid & 31;
    const int cg = blockIdx.y;

    for (int i = tid; i < a.Cin * 27 * CT; i += 128) {
        const int c = i % CT, r = i / CT;                   // r = ci*27 + tap
        s_w[i] = __ldg(a.w + (size_t)(cg * CT + c) * a.Cin * 27 + r);
    }
    if (!IDENT) load_norm(a.in0, a.Cin, s_sc, s_sh, tid, 128);
    
    __syncthreads();

    const int nsx = (a.Wout + 3) >> 2;
    const long long nstrips = (long long)a.Dout * a.Hout * nsx;
    const long long sid = (long long)blockIdx.x * 128 + tid;
    const bool active = sid < nstrips;
    int z = 0, y = 0, sx = 0;
    if (active) { sx = (int)(sid % nsx); long long r = sid / nsx; y = (int)(r % a.Hout); z = (int)(r / a.Hout); }
    const int x0 = sx * 4;                                   // first output x
    const int xin = x0 * STRIDE;                             // first centre input x
    const bool vec = (a.Win & 3) == 0;
    const size_t iplane = (size_t)a.Hin * a.Win, ivol = iplane * a.Din;

    float acc[4][CT];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < CT; ++c) acc[i][c] = 0.f;

    // Rows are software-pipelined: the RAW values of row (ci, dz, dy)+1 are requested before row (ci, dz, dy) is
    // activated and consumed, so a warp always has one 16/32-byte load in flight behind its FMAs (the coarse
    // levels run ~2 warps per scheduler and were bound by exposed load latency).  Out-of-range taps must be
    // zero AFTER the activation (zero padding of the activated tensor), hence the validity masks.
    bool xok[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) xok[i] = xin + i < a.Win;
    auto row_ptr = [&](int ci, int dz, int dy, bool& ok) -> const float* {
        const int zi = z * STRIDE - 1 + dz, yi = y * STRIDE - 1 + dy;
        ok = active && (unsigned)zi < (unsigned)a.Din && (unsigned)yi < (unsigned)a.Hin;
        return a.in0.x + (size_t)ci * ivol + ((long long)zi * (long long)iplane + (long long)yi * a.Win) + xin;
    };
    auto fetch = [&](const float* p, int xo, bool ok) -> float4 {     // raw; never dereferences an invalid address
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ok) {
            if (vec && xok[xo + 3]) v = __ldg(reinterpret_cast<const float4*>(p + xo));
            else {
                if (xok[xo]) v.x = __ldg(p + xo);
                if (xok[xo + 1]) v.y = __ldg(p + xo + 1);
                if (xok[xo + 2]) v.z = __ldg(p + xo + 2);
                if (xok[xo + 3]) v.w = __ldg(p + xo + 3);
            }
        }
        return v;
    };
    const bool halo_l = lane == 0 && sx > 0;
    const bool halo_r = STRIDE == 1 && lane == 31 && sx < nsx - 1 && xin + 4 < a.Win;

    bool ok_n;
    const float* p_n = row_ptr(0, 0, 0, ok_n);
    float4 n0 = fetch(p_n, 0, ok_n), n1 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (STRIDE == 2) n1 = fetch(p_n, 4, ok_n);
    for (int ci = 0; ci < a.Cin; ++ci) {
        const float sc0 = IDENT ? 1.f : s_sc[ci], sh0 = IDENT ? 0.f : s_sh[ci];
#pragma unroll
        for (int dz = 0; dz < 3; ++dz) {
#pragma unroll
            for (int dy = 0; dy < 3; ++dy) {
                const float4 r0 = n0, r1 = n1;
                const bool row_ok = ok_n;
                const float* p = p_n;
                {
                    const int dy2 = (dy + 1) % 3, dz2 = dy == 2 ? (dz + 1) % 3 : dz;
                    const bool wrap = dy == 2 && dz == 2;
                    p_n = row_ptr(wrap ? ci + 1 : ci, dz2, dy2, ok_n);
                    if (wrap && ci + 1 == a.Cin) ok_n = false;
                    n0 = fetch(p_n, 0, ok_n);
                    if (STRIDE == 2) n1 = fetch(p_n, 4, ok_n);
                }
                float hl = 0.f, hr = 0.f;
                if (halo_l && row_ok) hl = IDENT ? __ldg(p - 1) : act(__ldg(p - 1), sc0, sh0);
                if (halo_r && row_ok) hr = IDENT ? __ldg(p + 4) : act(__ldg(p + 4), sc0, sh0);
                // v[0] = input at xin-1, v[1..] = inputs at xin, xin+1, ...
                float v[STRIDE == 1 ? 6 : 9];
                v[1] = (IDENT || !(row_ok && xok[0])) ? r0.x : act(r0.x, sc0, sh0);
                v[2] = (IDENT || !(row_ok && xok[1])) ? r0.y : act(r0.y, sc0, sh0);
                v[3] = (IDENT || !(row_ok && xok[2])) ? r0.z : act(r0.z, sc0, sh0);
                v[4] = (IDENT || !(row_ok && xok[3])) ? r0.w : act(r0.w, sc0, sh0);
                float last = v[4];
                if (STRIDE == 2) {
                    v[5] = (IDENT || !(row_ok && xok[4])) ? r1.x : act(r1.x, sc0, sh0);
                    v[6] = (IDENT || !(row_ok && xok[5])) ? r1.y : act(r1.y, sc0, sh0);
                    v[7] = (IDENT || !(row_ok && xok[6])) ? r1.z : act(r1.z, sc0, sh0);
                    v[8] = (IDENT || !(row_ok && xok[7])) ? r1.w : act(r1.w, sc0, sh0);
                    last = v[8];
                }
                // halo from the neighbouring strips (same row when sx > 0 / sx < nsx-1)
                const float sl = __shfl_up_sync(0xffffffffu, last, 1);
                v[0] = (lane == 0 || sx == 0) ? hl : sl;
                if (STRIDE == 1) {
                    const float sr = __shfl_down_sync(0xffffffffu, v[1], 1);
                    v[5] = (lane == 31 || sx == nsx - 1) ? hr : sr;
                }
                const float* wrow = s_w + ((ci * 27) + dz * 9 + dy * 3) * CT;
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    float wv[CT];
#pragma unroll
                    for (int c4 = 0; c4 < CT / 4; ++c4) {
                        const float4 t = *reinterpret_cast<const float4*>(wrow + dx * CT + c4 * 4);
                        wv[c4 * 4] = t.x; wv[c4 * 4 + 1] = t.y; wv[c4 * 4 + 2] = t.z; wv[c4 * 4 + 3] = t.w;
                    }
#pragma unroll
                    for (int o = 0; o < 4; ++o) {
                        const float in = v[o * STRIDE + dx];
#pragma unroll
                        for (int c = 0; c < CT; ++c) acc[o][c] = fmaf(in, wv[c], acc[o][c]);
                    }
                }
            }
        }
    }
    store_and_stats<CT>(a, acc, active, z, y, x0, cg, s_stat, tid);
}

// ------------------------------------------------------------------------------------------
// conv0 (41 -> 8 on the raw cost volume, 60 % of CostRegNet's FLOPs): register-tiled variant.
// A thread owns 4 (x) x 2 (y) output voxels x 8 channels, so the four input rows y0-1 .. y0+2 of a
// depth slice feed both output rows (12 row loads instead of 18 per input channel) and every
// weight LDS.128 is amortised over 8 voxels.  Requires W % 4 == 0 and H % 2 == 0 (always true
// at level 0: D, H, W are multiples of 8) -- no scalar / dual-source / normalise paths are compiled
// in, which removes ~3/4 of the generic kernel's instruction stream.  The next row's 16-byte load is
// issued before the current row's 192 FMAs.  Accumulation order per output (ci, dz, dy, dx
// ascending) is the generic kernel's, so results are bit-identical to it.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128, 4)
conv0_k3_kernel(const ConvArgs a) {
    constexpr int CT = 8;
    extern __shared__ __align__(16) float s_w[];            // [Cin][27][8]
    __shared__ float s_stat[4 * 2 * CT];            // per-warp partial sums (4 warps), combined in fixed point
    const int tid = threadIdx.x, lane = tid & 31;

    for (int i = tid; i < a.Cin * 27 * CT; i += 128) {
        const int c = i % CT, r = i / CT;
        s_w[i] = __ldg(a.w + (size_t)c * a.Cin * 27 + r);
    }
    
    __syncthreads();

    const int W = a.Win, H = a.Hin, D = a.Din;
    const int nsx = W >> 2, H2 = H >> 1;
    const long long nstrips = (long long)D * H2 * nsx;
    const long long sid = (long long)blockIdx.x * 128 + tid;
    const bool active = sid < nstrips;
    int z = 0, y0 = 0, sx = 0;
    if (active) { sx = (int)(sid % nsx); long long r = sid / nsx; y0 = 2 * (int)(r % H2); z = (int)(r / H2); }
    const int x0 = sx * 4;
    const size_t iplane = (size_t)H * W, ivol = iplane * D;
    const bool first = sx == 0, last = sx == nsx - 1;

    // Row r (0..3) of the (ci, dz) slab is input row y0 - 1 + r at depth z - 1 + dz.  Offsets are 32-bit
    // (the launcher checks Cin * D * H * W < 2^31); validity is a 3-bit depth mask and a 4-bit row mask.
    const float* __restrict__ in = a.in0.x;
    const int iplane_i = (int)iplane, ivol_i = (int)ivol;
    const int off0 = (z - 1) * iplane_i + (y0 - 1) * W + x0;
    unsigned zmask = 0, ymask = 0;
    if (active) {
#pragma unroll
        for (int dz = 0; dz < 3; ++dz) zmask |= ((unsigned)(z - 1 + dz) < (unsigned)D) << dz;
#pragma unroll
        for (int r = 0; r < 4; ++r) ymask |= ((unsigned)(y0 - 1 + r) < (unsigned)H) << r;
    }
    const bool halo_l = lane == 0 && !first, halo_r = lane == 31 && !last;   // neighbours that are not in this warp

    float acc[2][4][CT];
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int c = 0; c < CT; ++c) acc[j][i][c] = 0.f;

    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 nxt = (zmask & 1u) && (ymask & 1u) ? __ldg(reinterpret_cast<const float4*>(in + off0)) : zero4;
    for (int ci = 0; ci < a.Cin; ++ci) {
        const int off_ci = off0 + ci * ivol_i;
#pragma unroll
        for (int dz = 0; dz < 3; ++dz) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const float4 cur = nxt;
                const int off = off_ci + dz * iplane_i + r * W;
                const bool ok = ((zmask >> dz) & 1u) && ((ymask >> r) & 1u);
                {   // prefetch the following row (wraps into the next dz / ci; after the last row, nothing)
                    const int r2 = (r + 1) & 3, dz2 = r == 3 ? (dz + 1) % 3 : dz;
                    const bool wrap = r == 3 && dz == 2;
                    const int off2 = off_ci + (wrap ? ivol_i : 0) + dz2 * iplane_i + r2 * W;
                    const bool ok2 = ((zmask >> dz2) & 1u) && ((ymask >> r2) & 1u) && !(wrap && ci + 1 == a.Cin);
                    nxt = zero4;
                    if (ok2) nxt = __ldg(reinterpret_cast<const float4*>(in + off2));
                }
                float hl = 0.f, hr = 0.f;
                if (halo_l && ok) hl = __ldg(in + off - 1);
                if (halo_r && ok) hr = __ldg(in + off + 4);
                const float sl = __shfl_up_sync(0xffffffffu, cur.w, 1);
                const float sr = __shfl_down_sync(0xffffffffu, cur.x, 1);
                float v[6];
                v[0] = (lane == 0 || first) ? hl : sl;
                v[1] = cur.x; v[2] = cur.y; v[3] = cur.z; v[4] = cur.w;
                v[5] = (lane == 31 || last) ? hr : sr;
#pragma unroll
                for (int j = 0; j < 2; ++j) {               // output row y0 + j sees this input row as tap dy = r - j
                    const int dy = r - j;
                    if (dy < 0 || dy > 2) continue;
                    const float* wrow = s_w + ((ci * 27) + dz * 9 + dy * 3) * CT;
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        const float4 w0 = *reinterpret_cast<const float4*>(wrow + dx * CT);
                        const float4 w1 = *reinterpret_cast<const float4*>(wrow + dx * CT + 4);
                        const float wv[CT] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                        for (int o = 0; o < 4; ++o) {
                            const float xin = v[o + dx];
#pragma unroll
                            for (int c = 0; c < CT; ++c) acc[j][o][c] = fmaf(xin, wv[c], acc[j][o][c]);
                        }
                    }
                }
            }
        }
    }

    const size_t plane = (size_t)a.Hout * a.Wout, vol = plane * a.Dout;
#pragma unroll
    for (int c = 0; c < CT; ++c) {
        float s = 0.f, q = 0.f;
        if (active) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                float* o = a.out + (size_t)c * vol + (size_t)z * plane + (size_t)(y0 + j) * a.Wout + x0;
                *reinterpret_cast<float4*>(o) = make_float4(acc[j][0][c], acc[j][1][c], acc[j][2][c], acc[j][3][c]);
#pragma unroll
                for (int i = 0; i < 4; ++i) { s += acc[j][i][c]; q = fmaf(acc[j][i][c], acc[j][i][c], q); }
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, off);
            q += __shfl_xor_sync(0xffffffffu, q, off);
        }
        if (lane == 0) { s_stat[(tid >> 5) * 2 * CT + 2 * c] = s; s_stat[(tid >> 5) * 2 * CT + 2 * c + 1] = q; }
    }
    __syncthreads();
    if (tid < 2 * CT)
        atomicAdd(reinterpret_cast<unsigned long long*>(a.stats_out) + tid,
                  stat_fx(s_stat[tid]) + stat_fx(s_stat[2 * CT + tid]) + stat_fx(s_stat[4 * CT + tid]) + stat_fx(s_stat[6 * CT + tid]));
}

// ------------------------------------------------------------------------------------------
// ConvTranspose3d k3 s2 p1 output_padding 1:  out[o] += in[i] * W[k],  o = 2 i - 1 + k, Dout = 2 Din.
// Sub-pixel decomposition: per axis, output 2i takes (k=1, in i); output 2i+1 takes (k=2, in i) and
// (k=0, in i+1).  So the 2x2x2 output block of input voxel (iz,iy,ix) depends on the 2x2x2 inputs
// (i .. i+1)^3 and uses each of the 27 taps exactly once: a thread owns one input voxel's output
// block x 8 channels (64 accumulators), every thread does the same 27 x 8 FMAs per input channel -- no
// parity divergence, no wasted taps.  Lanes are consecutive ix: the x+1 neighbour comes by shuffle, the
// 8 output rows are written as float2 (256 B per warp and row).  Two sources (U-Net skip sums) are
// activated separately and added on load; the next channel's loads are issued before the current FMAs.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
deconv3d_subpixel_kernel(const ConvArgs a) {
    constexpr int CT = 8;
    extern __shared__ __align__(16) float s_w[];            // [Cin][27][CT]
    __shared__ float s_sc[2][kMaxCin], s_sh[2][kMaxCin];
    __shared__ float s_stat[4 * 2 * CT];            // per-warp partial sums (4 warps), combined in fixed point
    const int tid = threadIdx.x, lane = tid & 31;
    const int cg = blockIdx.y;
    const bool dual = a.in1.x != nullptr;

    for (int i = tid; i < a.Cin * 27 * CT; i += 128) {
        const int c = i % CT, r = i / CT, ci = r / 27, tap = r - ci * 27;
        s_w[i] = __ldg(a.w + ((size_t)ci * a.Cout + cg * CT + c) * 27 + tap);
    }
    load_norm(a.in0, a.Cin, s_sc[0], s_sh[0], tid, 128);
    if (dual) load_norm(a.in1, a.Cin, s_sc[1], s_sh[1], tid, 128);
    
    __syncthreads();

    const long long nin = (long long)a.Din * a.Hin * a.Win;
    const long long vid = (long long)blockIdx.x * 128 + tid;
    const bool active = vid < nin;
    int iz = 0, iy = 0, ix = 0;
    if (active) { ix = (int)(vid % a.Win); long long r = vid / a.Win; iy = (int)(r % a.Hin); iz = (int)(r / a.Hin); }
    const size_t iplane = (size_t)a.Hin * a.Win, ivol = iplane * a.Din;
    const bool zok = iz + 1 < a.Din, yok = iy + 1 < a.Hin, xok = ix + 1 < a.Win;
    // the four (dz, dy) rows of this thread's own x column; [j] = dz * 2 + dy
    bool rok[4] = {active, active && yok, active && zok, active && zok && yok};
    size_t roff[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) roff[j] = (size_t)(iz + (j >> 1)) * iplane + (size_t)(iy + (j & 1)) * a.Win + ix;
    const bool need_r = lane == 31 && xok;                  // x+1 neighbour is not in this warp

    float acc[8][CT];                                        // [pz*4 + py*2 + px][c]
#pragma unroll
    for (int o = 0; o < 8; ++o)
#pragma unroll
        for (int c = 0; c < CT; ++c) acc[o][c] = 0.f;

    float n0[4], n1[4], r0[4], r1[4];                        // raw prefetch: own column / lane 31's right column
    auto fetch = [&](int ci) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            n0[j] = n1[j] = r0[j] = r1[j] = 0.f;
            if (rok[j]) {
                n0[j] = __ldg(a.in0.x + (size_t)ci * ivol + roff[j]);
                if (dual) n1[j] = __ldg(a.in1.x + (size_t)ci * ivol + roff[j]);
                if (need_r) {
                    r0[j] = __ldg(a.in0.x + (size_t)ci * ivol + roff[j] + 1);
                    if (dual) r1[j] = __ldg(a.in1.x + (size_t)ci * ivol + roff[j] + 1);
                }
            }
        }
    };
    fetch(0);
    for (int ci = 0; ci < a.Cin; ++ci) {
        const float sc0 = s_sc[0][ci], sh0 = s_sh[0][ci];
        const float sc1 = dual ? s_sc[1][ci] : 1.f, sh1 = dual ? s_sh[1][ci] : 0.f;
        float in[4][2];                                      // [dz*2+dy][dx], activated, zero outside the tensor
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float v = 0.f, vr = 0.f;
            if (rok[j]) {
                v = act(n0[j], sc0, sh0);
                if (dual) v += act(n1[j], sc1, sh1);
                if (need_r) { vr = act(r0[j], sc0, sh0); if (dual) vr += act(r1[j], sc1, sh1); }
            }
            const float sh = __shfl_down_sync(0xffffffffu, v, 1);
            in[j][0] = v;
            in[j][1] = !xok ? 0.f : (lane == 31 ? vr : sh);
        }
        if (ci + 1 < a.Cin) fetch(ci + 1);
        const float* wci = s_w + (size_t)ci * 27 * CT;
        // per axis the three (d, p, k) combinations: (0,0,1) (0,1,2) (1,1,0)
#pragma unroll
        for (int az = 0; az < 3; ++az) {
            const int dz = az == 2, pz = az != 0, kz = az == 0 ? 1 : (az == 1 ? 2 : 0);
#pragma unroll
            for (int ay = 0; ay < 3; ++ay) {
                const int dy = ay == 2, py = ay != 0, ky = ay == 0 ? 1 : (ay == 1 ? 2 : 0);
#pragma unroll
                for (int ax = 0; ax < 3; ++ax) {
                    const int dx = ax == 2, px = ax != 0, kx = ax == 0 ? 1 : (ax == 1 ? 2 : 0);
                    const float* wp = wci + (kz * 9 + ky * 3 + kx) * CT;
                    const float4 w0 = *reinterpret_cast<const float4*>(wp);
                    const float4 w1 = *reinterpret_cast<const float4*>(wp + 4);
                    const float wv[CT] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
                    const float x = in[dz * 2 + dy][dx];
                    const int o = pz * 4 + py * 2 + px;
#pragma unroll
                    for (int c = 0; c < CT; ++c) acc[o][c] = fmaf(x, wv[c], acc[o][c]);
                }
            }
        }
    }

    const size_t plane = (size_t)a.Hout * a.Wout, vol = plane * a.Dout;
#pragma unroll
    for (int c = 0; c < CT; ++c) {
        float s = 0.f, q = 0.f;
        if (active) {
            float* o = a.out + (size_t)(cg * CT + c) * vol + (size_t)(2 * iz) * plane + (size_t)(2 * iy) * a.Wout + 2 * ix;
#pragma unroll
            for (int j = 0; j < 4; ++j) {                   // j = pz*2 + py
                *reinterpret_cast<float2*>(o + (size_t)(j >> 1) * plane + (size_t)(j & 1) * a.Wout) =
                    make_float2(acc[j * 2][c], acc[j * 2 + 1][c]);
                s += acc[j * 2][c] + acc[j * 2 + 1][c];
                q = fmaf(acc[j * 2][c], acc[j * 2][c], q);
                q = fmaf(acc[j * 2 + 1][c], acc[j * 2 + 1][c], q);
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, off);
            q += __shfl_xor_sync(0xffffffffu, q, off);
        }
        if (lane == 0) { s_stat[(tid >> 5) * 2 * CT + 2 * c] = s; s_stat[(tid >> 5) * 2 * CT + 2 * c + 1] = q; }
    }
    __syncthreads();
    if (tid < 2 * CT)       // four warp partials -> fixed point -> ONE integer atomic per CTA and slot (order-independent)
        atomicAdd(reinterpret_cast<unsigned long long*>(a.stats_out) + 2 * (cg * CT) + tid,
                  stat_fx(s_stat[tid]) + stat_fx(s_stat[2 * CT + tid]) + stat_fx(s_stat[4 * CT + tid]) + stat_fx(s_stat[6 * CT + tid]));
}

// ------------------------------------------------------------------------------------------
// final: volume = ABN(conv0) + ABN(deconv11)  -> channels-last [nvox][8]   (models.py:766)
// F16: the fp32 sums rounded with __float2half_rn, one 16-byte store of eight halves per voxel
// ------------------------------------------------------------------------------------------
template <bool F16>
__global__ void __launch_bounds__(256)
finalize_volume_kernel(ActSrc s0, ActSrc s1, long long nvox, float4* __restrict__ out) {
    __shared__ float sc[2][8], sh[2][8];
    load_norm(s0, 8, sc[0], sh[0], threadIdx.x, 256);
    load_norm(s1, 8, sc[1], sh[1], threadIdx.x, 256);
    __syncthreads();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox; i += (long long)gridDim.x * blockDim.x) {
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c)
            v[c] = act(__ldg(s0.x + c * nvox + i), sc[0][c], sh[0][c]) + act(__ldg(s1.x + c * nvox + i), sc[1][c], sh[1][c]);
        if constexpr (F16) {
            uint32_t h[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                h[j] = (uint32_t)__half_as_ushort(__float2half_rn(v[2 * j])) |
                       ((uint32_t)__half_as_ushort(__float2half_rn(v[2 * j + 1])) << 16);
            reinterpret_cast<uint4*>(out)[i] = make_uint4(h[0], h[1], h[2], h[3]);
        } else {
            out[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
            out[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
        }
    }
}

// ------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------
struct Dims { int D, H, W; long long n() const { return (long long)D * H * W; } };

template <int CT, int STRIDE, bool IDENT>
static int launch_conv(const ConvArgs& a, cudaStream_t st) {
    const size_t smem = (size_t)a.Cin * 27 * CT * sizeof(float);
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(conv3d_k3_kernel<CT, STRIDE, IDENT>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long nstrips = (long long)a.Dout * a.Hout * ((a.Wout + 3) / 4);
    dim3 grid(cdiv(nstrips, 128), a.Cout / CT);
    conv3d_k3_kernel<CT, STRIDE, IDENT><<<grid, 128, smem, st>>>(a);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

static int launch_conv0(const ConvArgs& a, cudaStream_t st) {
    if (a.Cout != 8 || (a.Win & 3) || (a.Hin & 1) || (long long)a.Cin * a.Din * a.Hin * a.Win >= (1ll << 31))
        return launch_conv<8, 1, true>(a, st);
    const size_t smem = (size_t)a.Cin * 27 * 8 * sizeof(float);
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(conv0_k3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long nstrips = (long long)a.Dout * (a.Hout / 2) * (a.Wout / 4);
    conv0_k3_kernel<<<(unsigned)cdiv(nstrips, 128), 128, smem, st>>>(a);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

// Coarse levels have few voxels (level 3 of a 128x176x208 volume: 9152): narrow the per-CTA output-channel
// tile until the grid covers the SMs about twice (the layers are latency-, not throughput-bound there).
template <int STRIDE>
static int launch_conv_auto(const ConvArgs& a, cudaStream_t st) {
    const long long ctas16 = cdiv((long long)a.Dout * a.Hout * ((a.Wout + 3) / 4), 128) * (a.Cout / 16);
    const int want = 2 * sm_count();
    if (ctas16 >= want || a.Cout % 16) return launch_conv<16, STRIDE, false>(a, st);
    if (ctas16 * 2 >= want) return launch_conv<8, STRIDE, false>(a, st);
    return launch_conv<4, STRIDE, false>(a, st);
}

static int launch_deconv(const ConvArgs& a, cudaStream_t st) {
    const size_t smem = (size_t)a.Cin * 27 * 8 * sizeof(float);
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(deconv3d_subpixel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long nin = (long long)a.Din * a.Hin * a.Win;
    dim3 grid(cdiv(nin, 128), a.Cout / 8);
    deconv3d_subpixel_kernel<<<grid, 128, smem, st>>>(a);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

__global__ void bn_update_running_kernel(BnUpdateArgs a) {
    const int l = blockIdx.x, c = threadIdx.x;
    if (c >= a.C[l]) return;
    const double count = a.count[l];
    const double mean = stat_value(a.stats[l] + 2 * c) / count;
    double var = stat_value(a.stats[l] + 2 * c + 1) / count - mean * mean;
    var = var > 0.0 ? var : 0.0;
    const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    const double m = (double)a.momentum;
    a.rmean[l][c] = (float)((1.0 - m) * (double)a.rmean[l][c] + m * mean);
    a.rvar[l][c] = (float)((1.0 - m) * (double)a.rvar[l][c] + m * unbiased);
}

}  // namespace mvsn

using namespace mvsn;

// layer table: conv0..conv6 (Conv3d), conv7/9/11 (ConvTranspose3d)
static const int kCin[10]  = {41, 8, 16, 16, 32, 32, 64, 64, 32, 16};
static const int kCout[10] = {8, 16, 16, 32, 32, 64, 64, 32, 16, 8};
static const int kLevelOut[10] = {0, 1, 1, 2, 2, 3, 3, 2, 1, 0};     // resolution level of each layer's output

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static int costreg_forward(const float* const* w, float* const* running, int bn_mode, float momentum, const float* cost,
                           int D, int Hp, int Wp, void* volume_dhwc, bool f16, void* workspace, size_t workspace_bytes,
                           void* stream_);

extern "C" {

size_t mvsn_costreg_workspace_bytes(int D, int Hp, int Wp) {
    size_t total = 4096;                                       // statistics block (10 layers x <=64 ch x 2 doubles)
    total += 10 * 64 * 2 * sizeof(double);
    total += align_up(conv0_tc_workspace_bytes(), 4096);        // conv0's tensor-core weight image (hi | lo)
    for (int l = 0; l < 10; ++l) {
        const int s = 1 << kLevelOut[l];
        total += align_up((size_t)kCout[l] * (D / s) * (Hp / s) * (Wp / s) * sizeof(float), 256);
    }
    return total;
}

int mvsn_costreg_forward(const float* const* w, const float* cost, int D, int Hp, int Wp, float* volume_dhwc,
                         void* workspace, size_t workspace_bytes, void* stream_) {
    return mvsn_costreg_forward_bn(w, nullptr, MVSN_BN_BATCH, 0.f, cost, D, Hp, Wp, volume_dhwc, workspace, workspace_bytes, stream_);
}

int mvsn_costreg_forward_bn(const float* const* w, float* const* running, int bn_mode, float momentum, const float* cost,
                            int D, int Hp, int Wp, float* volume_dhwc, void* workspace, size_t workspace_bytes, void* stream_) {
    MVSN_RANGE("mvsn_costreg_forward_bn");
    return costreg_forward(w, running, bn_mode, momentum, cost, D, Hp, Wp, volume_dhwc, false, workspace, workspace_bytes,
                           stream_);
}

int mvsn_costreg_forward_f16(const float* const* w, float* const* running, int bn_mode, float momentum, const float* cost,
                             int D, int Hp, int Wp, void* volume_dhwc_f16, void* workspace, size_t workspace_bytes,
                             void* stream_) {
    MVSN_RANGE("mvsn_costreg_forward_f16");
    return costreg_forward(w, running, bn_mode, momentum, cost, D, Hp, Wp, volume_dhwc_f16, true, workspace,
                           workspace_bytes, stream_);
}

}  // extern "C"

// mvsn_costreg_forward_bn (f16 = false: fp32 volume) and mvsn_costreg_forward_f16
static int costreg_forward(const float* const* w, float* const* running, int bn_mode, float momentum, const float* cost,
                           int D, int Hp, int Wp, void* volume_dhwc, bool f16, void* workspace, size_t workspace_bytes,
                           void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    const bool conv0_ffma_flag = (bn_mode & MVSN_CONV0_FFMA) != 0;
    bn_mode &= ~MVSN_CONV0_FFMA;
    MVSN_REQUIRE(bn_mode == MVSN_BN_BATCH || bn_mode == MVSN_BN_BATCH_UPDATE || bn_mode == MVSN_BN_RUNNING, MVSN_EBADSHAPE,
                 "mvsn_costreg_forward_bn: bn_mode %d", bn_mode);
    MVSN_REQUIRE(bn_mode == MVSN_BN_BATCH || running, MVSN_ENULL, "mvsn_costreg_forward_bn: running statistics are NULL");
    if (bn_mode != MVSN_BN_BATCH)
        for (int i = 0; i < 20; ++i) MVSN_REQUIRE(running[i] != nullptr, MVSN_ENULL, "mvsn_costreg_forward_bn: running[%d] is NULL", i);
    MVSN_REQUIRE(w && cost && volume_dhwc && workspace, MVSN_ENULL, "mvsn_costreg_forward: NULL argument");
    MVSN_REQUIRE(D > 0 && Hp > 0 && Wp > 0 && D % 8 == 0 && Hp % 8 == 0 && Wp % 8 == 0, MVSN_EBADSHAPE,
                 "mvsn_costreg_forward: D=%d Hp=%d Wp=%d must all be divisible by 8 (three stride-2 levels, models.py:730-766)",
                 D, Hp, Wp);
    MVSN_REQUIRE(workspace_bytes >= mvsn_costreg_workspace_bytes(D, Hp, Wp), MVSN_EWORKSPACE,
                 "mvsn_costreg_forward: workspace too small");
    MVSN_REQUIRE(aligned16(workspace) && aligned16(volume_dhwc) && aligned16(cost), MVSN_EALIGN,
                 "mvsn_costreg_forward: buffers must be 16-byte aligned");
    for (int i = 0; i < MVSN_N_COSTREG_TENSORS; ++i)
        MVSN_REQUIRE(w[i] != nullptr, MVSN_ENULL, "mvsn_costreg_forward: weight %d is NULL", i);

    // carve the workspace
    char* p = static_cast<char*>(workspace);
    double* stats = reinterpret_cast<double*>(p);
    const size_t stats_bytes = 10 * 64 * 2 * sizeof(double);
    p += align_up(stats_bytes, 4096);
    void* conv0_wimg = p;
    p += align_up(conv0_tc_workspace_bytes(), 4096);
    float* raw[10];
    Dims dims[10];
    for (int l = 0; l < 10; ++l) {
        const int s = 1 << kLevelOut[l];
        dims[l] = {D / s, Hp / s, Wp / s};
        raw[l] = reinterpret_cast<float*>(p);
        p += align_up((size_t)kCout[l] * dims[l].n() * sizeof(float), 256);
    }
    MVSN_CUDA_CHECK(cudaMemsetAsync(stats, 0, stats_bytes, st));

    auto src = [&](int l) {
        ActSrc s;
        s.x = raw[l]; s.stats = stats + (size_t)l * 128; s.gamma = w[3 * l + 1]; s.beta = w[3 * l + 2];
        s.count = (double)dims[l].n();
        s.rmean = bn_mode == MVSN_BN_RUNNING ? running[2 * l] : nullptr;
        s.rvar = bn_mode == MVSN_BN_RUNNING ? running[2 * l + 1] : nullptr;
        return s;
    };
    const ActSrc none{nullptr, nullptr, nullptr, nullptr, 1.0, nullptr, nullptr};
    auto args = [&](int l, ActSrc a0, ActSrc a1, Dims din) {
        ConvArgs a;
        a.in0 = a0; a.in1 = a1; a.Cin = kCin[l]; a.Din = din.D; a.Hin = din.H; a.Win = din.W;
        a.w = w[3 * l]; a.Cout = kCout[l]; a.Dout = dims[l].D; a.Hout = dims[l].H; a.Wout = dims[l].W;
        a.out = raw[l]; a.stats_out = stats + (size_t)l * 128;
        return a;
    };
    int rc;
    ActSrc cost_src{cost, nullptr, nullptr, nullptr, 1.0, nullptr, nullptr};
    const Dims full{D, Hp, Wp};
    // conv0 41->8: wgmma kernel (conv0_tc.cu); the MVSN_CONV0_FFMA flag (or MVSN_CONV0=ffma in the environment) selects
    // the round-1 FFMA kernel for A/B comparisons
    static const bool conv0_ffma_env = [] { const char* e = getenv("MVSN_CONV0"); return e && !strcmp(e, "ffma"); }();
    if (conv0_ffma_env || conv0_ffma_flag) rc = launch_conv0(args(0, cost_src, none, full), st);
    else rc = launch_conv0_tc(args(0, cost_src, none, full), conv0_wimg, st);
    if (rc) return rc;
    if ((rc = launch_conv_auto<2>(args(1, src(0), none, dims[0]), st))) return rc;       // conv1 8->16 s2
    if ((rc = launch_conv_auto<1>(args(2, src(1), none, dims[1]), st))) return rc;       // conv2 16->16
    if ((rc = launch_conv_auto<2>(args(3, src(2), none, dims[2]), st))) return rc;       // conv3 16->32 s2
    if ((rc = launch_conv_auto<1>(args(4, src(3), none, dims[3]), st))) return rc;       // conv4 32->32
    if ((rc = launch_conv_auto<2>(args(5, src(4), none, dims[4]), st))) return rc;       // conv5 32->64 s2
    if ((rc = launch_conv_auto<1>(args(6, src(5), none, dims[5]), st))) return rc;       // conv6 64->64
    if ((rc = launch_deconv(args(7, src(6), none, dims[6]), st))) return rc;               // conv7  64->32
    if ((rc = launch_deconv(args(8, src(4), src(7), dims[7]), st))) return rc;             // conv9  (conv4 + .) 32->16
    if ((rc = launch_deconv(args(9, src(2), src(8), dims[8]), st))) return rc;              // conv11 (conv2 + .) 16->8
    const long long nvox = full.n();
    const int fgrid = cdiv(nvox, 256) < sm_count() * 8 ? cdiv(nvox, 256) : sm_count() * 8;
    if (f16) finalize_volume_kernel<true><<<fgrid, 256, 0, st>>>(src(0), src(9), nvox, reinterpret_cast<float4*>(volume_dhwc));
    else     finalize_volume_kernel<false><<<fgrid, 256, 0, st>>>(src(0), src(9), nvox, reinterpret_cast<float4*>(volume_dhwc));
    MVSN_CUDA_CHECK(cudaGetLastError());
    if (bn_mode == MVSN_BN_BATCH_UPDATE) {
        BnUpdateArgs u{};
        for (int l = 0; l < 10; ++l) {
            u.stats[l] = stats + (size_t)l * 128; u.count[l] = (double)dims[l].n(); u.C[l] = kCout[l];
            u.rmean[l] = running[2 * l]; u.rvar[l] = running[2 * l + 1];
        }
        u.momentum = momentum;
        bn_update_running_kernel<<<10, 64, 0, st>>>(u);
    }
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}
