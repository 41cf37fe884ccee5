// Per-sample front end of the fused render kernel: everything the reference does between
// "a ray" and "the 86-channel MLP input" (renderer.py:138-165 and callees), as device functions
// shared by the fp32 and the tensor-core (wgmma) render kernels.
#pragma once
#include <cuda_fp16.h>
#include <type_traits>
#include "common.cuh"

namespace mvsn {

struct SceneDev {
    const float* vol;      // [D,Hp,Wp,8]; fp16 halves (read as such) in the half-volume render instantiations
    const float4* imgs;    // [V,H,W] texels (r,g,b,0)
    int D, Hp, Wp;
    int V, H, W;
    const float* w2cs;     // [V,4,4] device
    const float* intrinsics;  // [V,3,3] device
    int white_bkgd;
};

struct Cams {              // staged in shared memory by every render kernel
    float w2c[3][12];
    float K[3][9];
};

__device__ __forceinline__ void load_cams(const SceneDev& sc, Cams* cams, int tid) {
    if (tid < 36) cams->w2c[tid / 12][tid % 12] = __ldg(sc.w2cs + (tid / 12) * 16 + tid % 12);
    else if (tid < 63) { const int i = tid - 36; cams->K[i / 9][i % 9] = __ldg(sc.intrinsics + i); }
}

struct RayGenDev {
    float near, far_minus_near;      // z normalisation of the reference camera (utils.py:128-131)
    float inv_near, inv_far_minus_inv_near;
    float pad, wf, hf;               // utils.py:138-143
    int lindisp;
};

struct RenderIO {
    // signature-compatible inputs (FAST == false)
    const float* pts; const float* ndc; const float* z; const float* dirs;
    // fused-caller inputs (FAST == true)
    const float* rays; const float* t_steps;
    RayGenDev rg;
    int N, S;
    int rays_per_tile;     // tensor-core kernel: chosen by its launcher
    float* rgb; float* depth; float* weights; float* alpha; float* input_feat;
    // multi-GPU frame sink (mvsn_render_rays_to_peers): every finished pixel is stored as one 16-byte
    // (r, g, b, depth) texel into EVERY rank's copy of the assembled frame, straight from the compositing
    // epilogue over NVLink peer mappings -- the frame is complete on all ranks when the kernels are, with no
    // gather pass.  n_sink == 0: off.
    float4* sink[MVSN_MAX_PEERS];
    int n_sink;
    long long sink_first;  // frame index of this launch's ray 0
};

// final pixel of ray `ray`: the caller's rgb / depth arrays (either may be null when a sink is given) and the sink
__device__ __forceinline__ void store_pixel(const RenderIO& io, int ray, float r, float g, float b, float d) {
    if (io.rgb) { io.rgb[(size_t)ray * 3 + 0] = r; io.rgb[(size_t)ray * 3 + 1] = g; io.rgb[(size_t)ray * 3 + 2] = b; }
    if (io.depth) io.depth[ray] = d;
    if (io.n_sink > 0) {
        const float4 px = make_float4(r, g, b, d);
        const long long at = io.sink_first + ray;
#pragma unroll 1
        for (int p = 0; p < io.n_sink; ++p) io.sink[p][at] = px;
    }
}

int launch_render_fp32(const SceneDev& sc, const RenderIO& io, bool fast, const float* wts, cudaStream_t stream);
// tensor-core modes (render_wg.cu): split = MVSN_MLP_TC_SPLIT, otherwise the fp16-operand modes.  t_stop != NULL
// (fast only): early ray termination at transmittance *t_stop; tiles_done (may be NULL) += the tiles computed.
// half_vol: sc.vol is an fp16 [D,Hp,Wp,8] image (MVSN_VOLUME_F16).  occ_bits (with t_stop; empty-space skipping): an
// occupancy grid of the scene's D x Hp x Wp cells; its per-group tile ranges go to `ranges` (occupancy_ranges_bytes(N)).
int launch_render_wg(const SceneDev& sc, const RenderIO& io, bool fast, bool split, const void* wimg, cudaStream_t stream,
                     const float* t_stop = nullptr, unsigned long long* tiles_done = nullptr, bool half_vol = false,
                     const uint32_t* occ_bits = nullptr, int2* ranges = nullptr);
// occupancy.cu: the grid (mvsn_build_occupancy; wimg_split = the MVSN_MLP_TC_SPLIT image) and the range pre-pass of a
// ray launch (io.rays_per_tile set; precise = the split mode's NDC arithmetic)
size_t occupancy_words(int D, int Hp, int Wp);
size_t occupancy_workspace_bytes(int D, int Hp, int Wp);
size_t occupancy_ranges_bytes(int N);
int build_occupancy(const SceneDev& sc, const RayGenDev& rg, const void* wimg_split, bool half_vol, int dilate,
                    uint32_t* bits, void* workspace, cudaStream_t stream);
int launch_occupancy_ranges(const SceneDev& sc, const RenderIO& io, bool precise, const uint32_t* bits, int2* ranges,
                            cudaStream_t stream);
// occupancy.cu: the density grid (mvsn_build_density): fp32 sigma [D][Hp][Wp] at the nodes, by the fp32 forward tile
size_t density_workspace_bytes(int D, int Hp, int Wp);
int build_density(const SceneDev& sc, const RayGenDev& rg, const float* wts_fp32, bool half_vol, float* sigma,
                  void* workspace, cudaStream_t stream);
// importance.cu: inverse-CDF sampling from a density grid (mvsn_sample_importance).  The coarse samples are marched
// from rays / t_steps / jitter (t_steps set) or read from z_in / ndc_in; cams: sc's cameras are valid (needed by the
// march and by ndc_out); sc.D / Hp / Wp are the grid's dims.
struct ImportanceIO {
    const float* rays; const float* t_steps; const float* jitter;
    const float* z_in; const float* ndc_in;
    const float* sigma; const float* u;
    int N, S, K, cams;
    float* z_out; float* pts_out; float* ndc_out;
};
constexpr int MAX_IMPORTANCE_SAMPLES = 1024;             // S + K
int launch_importance(const SceneDev& sc, const RayGenDev& rg, const ImportanceIO& io, cudaStream_t stream);
// fp16 [D,Hp,Wp,8] image of a planar [8,D,Hp,Wp] or channels-last volume, fp32 or fp16, rounded with __float2half_rn
int launch_volume_to_half(const void* src, bool src_half, bool src_planar, long long nvox, void* dst, cudaStream_t stream);
size_t mlp_wg_packed_bytes(bool split);
int pack_mlp_wg(const float* const* w, bool split, void* packed, cudaStream_t stream);
// fine-tuning step (render_bwd.cu); grad_mode: MVSN_MLP_FP32, MVSN_MLP_TC_HALF (dgrad / wgrad GEMMs on wgmma with
// fp16 operands) or MVSN_GRAD_TC_FULL (TC_HALF plus the forward recompute's GEMMs on wgmma; io.rays entries only);
// det: the volume gradient and the loss summed in a fixed order (bit-reproducible); io.rays set: the samples are
// marched in the kernel from io.rays / io.t_steps, stratified by `jitter` [N,S] (NULL: none), instead of read from
// io.pts / io.ndc / io.z / io.dirs
// backward_layout: byte offsets in one call's workspace (the grad mode's, then `det`'s and `stop`'s buffers); D = Hp =
// Wp = 0: a frozen volume.  total == 0: an unsupported shape or grad mode.
struct BwdLayout { size_t loss, amax, acc, rec, live, list, total; int list_cap; };
BwdLayout backward_layout(int N, int S, int D, int Hp, int Wp, int grad_mode, bool det, bool stop);
// early ray termination (the _stop entries); live_samples / tiles_done may be NULL
struct BwdStop { float t_stop; int* live_samples; unsigned long long* tiles_done; };
// one backward call, every argument but the workspace checked by the entry `what`; dvol NULL: a frozen volume
struct BwdCall {
    const char* what; const mvsn_render_grads* g; const float* const* mlp_w; float* const* grad_mlp; float* dvol;
    void* workspace; size_t workspace_bytes; int grad_mode; bool det; const float* jitter; const BwdStop* stop;
};
int launch_render_backward(const SceneDev& sc, const RenderIO& io, const float* wts_fp32, const BwdCall& call,
                           cudaStream_t stream);
int launch_adam_tensors(float* const* p, const float* const* g, float* const* m, float* const* v, const int* n, int count,
                        float lr, float beta1, float beta2, float eps, int step, cudaStream_t stream);
int launch_adam_volume(float* p, float* g_dhwc, float* m, float* v, long long nvox, int planar, float lr, float beta1,
                       float beta2, float eps, int step, cudaStream_t stream);

// cam = R p + t ; pix = K cam ; (u, v) = pix.xy / pix.z / (W-1, H-1)     utils.py:120-127
template <bool PRECISE>
__device__ __forceinline__ float fdiv(float a, float b) { return PRECISE ? __fdiv_rn(a, b) : __fdividef(a, b); }

// PRECISE = IEEE divisions exactly where the reference divides (fp32-parity modes); otherwise
// MUFU.RCP-based divisions (2 ulp), plenty for the 16-bit-operand mode and a fraction of the code.
template <bool PRECISE = true>
__device__ __forceinline__ void project_view(const float* __restrict__ w2c, const float* __restrict__ K,
                                             float px, float py, float pz, float wm1, float hm1,
                                             float& u, float& v, float& zc) {
    float cx = fmaf(pz, w2c[2], fmaf(py, w2c[1], px * w2c[0])) + w2c[3];
    float cy = fmaf(pz, w2c[6], fmaf(py, w2c[5], px * w2c[4])) + w2c[7];
    float cz = fmaf(pz, w2c[10], fmaf(py, w2c[9], px * w2c[8])) + w2c[11];
    float qx = fmaf(cz, K[2], fmaf(cy, K[1], cx * K[0]));
    float qy = fmaf(cz, K[5], fmaf(cy, K[4], cx * K[3]));
    float qz = fmaf(cz, K[8], fmaf(cy, K[7], cx * K[6]));
    if (PRECISE) {
        u = __fdiv_rn(__fdiv_rn(qx, qz), wm1);
        v = __fdiv_rn(__fdiv_rn(qy, qz), hm1);
    } else {
        const float iz = __fdividef(1.f, qz);
        u = qx * iz * __fdividef(1.f, wm1);
        v = qy * iz * __fdividef(1.f, hm1);
    }
    zc = qz;
}

// utils.get_ndc_coordinate for the reference camera (utils.py:112-146)
template <bool PRECISE = true>
__device__ __forceinline__ void ndc_of_point(const SceneDev& sc, const Cams& cams, const RayGenDev& rg,
                                             float px, float py, float pz,
                                             float& nx, float& ny, float& nz) {
    float u, v, zc;
    project_view<PRECISE>(cams.w2c[0], cams.K[0], px, py, pz, (float)(sc.W - 1), (float)(sc.H - 1), u, v, zc);
    if (!rg.lindisp) nz = fdiv<PRECISE>(zc - rg.near, rg.far_minus_near);
    else             nz = fdiv<PRECISE>(fdiv<PRECISE>(1.0f, zc) - rg.inv_near, rg.inv_far_minus_inv_near);
    if (rg.pad > 0.f) {
        float dh = rg.hf + rg.pad * 2.f, dw = rg.wf + rg.pad * 2.f;
        v = __fadd_rn(fdiv<PRECISE>(__fmul_rn(v, rg.hf), dh), fdiv<PRECISE>(rg.pad, dh));
        u = __fadd_rn(fdiv<PRECISE>(__fmul_rn(u, rg.wf), dw), fdiv<PRECISE>(rg.pad, dw));
    }
    nx = u; ny = v;
}

// ray-march depth at step t in [0, 1] (data/ray_utils.py:177-180), rounded as the reference's fp32 ops round
__device__ __forceinline__ float ray_z(float near, float far, float t, int lindisp) {
    if (!lindisp) return __fadd_rn(__fmul_rn(near, 1.f - t), __fmul_rn(far, t));
    return __fdiv_rn(1.f, __fadd_rn(__fmul_rn(__fdiv_rn(1.f, near), 1.f - t), __fmul_rn(__fdiv_rn(1.f, far), t)));
}

// stratified depth of sample s of S (data/ray_utils.py:184-191, perturb > 0): lower + (upper - lower) j, between the
// midpoints of the neighbouring ray_z depths (lower = z_0 for s = 0, upper = z_{S-1} for s = S - 1), j = perturb * u.
// Every operation rounded on its own, as ray_marcher's element-wise PyTorch ops round them.
__device__ __forceinline__ float ray_z_jittered(float near, float far, const float* t_steps, int s, int S, int lindisp,
                                                float j) {
    const float z = ray_z(near, far, __ldg(t_steps + s), lindisp);
    const float lower = s == 0 ? z : __fmul_rn(0.5f, __fadd_rn(ray_z(near, far, __ldg(t_steps + s - 1), lindisp), z));
    const float upper = s == S - 1 ? z : __fmul_rn(0.5f, __fadd_rn(z, ray_z(near, far, __ldg(t_steps + s + 1), lindisp)));
    return __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), j));
}

// ray-march point (px, py, pz), ray direction (dx, dy, dz), NDC (nx, ny, nz) and depth z of sample s_idx of ray `ray`:
// marched from io.rays / io.t_steps (FAST) or read from the caller's per-sample arrays (si = ray * S + s_idx).
// FAST with `jitter` ([N,S], the fine-tuning backward): the stratified depth ray_z_jittered with j = jitter[si].
template <bool FAST, bool PRECISE>
__device__ __forceinline__ void sample_point(const SceneDev& sc, const Cams& cams, const RenderIO& io, int ray, int s_idx,
                                             size_t si, float& px, float& py, float& pz, float& dx, float& dy, float& dz,
                                             float& nx, float& ny, float& nz, float& z, const float* jitter = nullptr) {
    if (FAST) {
        const float4* rp = reinterpret_cast<const float4*>(io.rays + (size_t)ray * 8);
        float4 r0 = __ldg(rp), r1 = __ldg(rp + 1);
        dx = r0.w; dy = r1.x; dz = r1.y;
        if (jitter) z = ray_z_jittered(r1.z, r1.w, io.t_steps, s_idx, io.S, io.rg.lindisp, __ldg(jitter + si));
        else        z = ray_z(r1.z, r1.w, __ldg(io.t_steps + s_idx), io.rg.lindisp);
        px = __fadd_rn(r0.x, __fmul_rn(dx, z));
        py = __fadd_rn(r0.y, __fmul_rn(dy, z));
        pz = __fadd_rn(r0.z, __fmul_rn(dz, z));
        ndc_of_point<PRECISE>(sc, cams, io.rg, px, py, pz, nx, ny, nz);
    } else {
        px = __ldg(io.pts + si * 3); py = __ldg(io.pts + si * 3 + 1); pz = __ldg(io.pts + si * 3 + 2);
        nx = __ldg(io.ndc + si * 3); ny = __ldg(io.ndc + si * 3 + 1); nz = __ldg(io.ndc + si * 3 + 2);
        z = io.z[si];                                   // plain load: removed where z is unused
        dx = __ldg(io.dirs + (size_t)ray * 3); dy = __ldg(io.dirs + (size_t)ray * 3 + 1);
        dz = __ldg(io.dirs + (size_t)ray * 3 + 2);
    }
}

// Trilinear footprint of an NDC point in the volume (utils.py:357-383, align_corners=True): the corner origin and the
// per-axis corner weights, with no masking.  Corner c = (x0 + (c & 1), y0 + ((c >> 1) & 1), z0 + (c >> 2)) has weight
// wx[c & 1] * wy[(c >> 1) & 1] * wz[c >> 2]; corners outside the volume are the caller's to handle.
struct Trilinear {
    int x0, y0, z0;
    float wx[2], wy[2], wz[2];
};
__device__ __forceinline__ Trilinear trilinear_corners(const SceneDev& sc, float nx, float ny, float nz) {
    const int W = sc.Wp, H = sc.Hp, D = sc.D;
    const float ix = ((nx * 2.f - 1.f + 1.f) * 0.5f) * (float)(W - 1);
    const float iy = ((ny * 2.f - 1.f + 1.f) * 0.5f) * (float)(H - 1);
    const float iz = ((nz * 2.f - 1.f + 1.f) * 0.5f) * (float)(D - 1);
    const float x0f = floorf(ix), y0f = floorf(iy), z0f = floorf(iz);
    Trilinear t;
    t.wx[0] = (x0f + 1.f) - ix; t.wx[1] = ix - x0f;
    t.wy[0] = (y0f + 1.f) - iy; t.wy[1] = iy - y0f;
    t.wz[0] = (z0f + 1.f) - iz; t.wz[1] = iz - z0f;
    // clamp before the int conversion so absurd coordinates cannot overflow
    t.x0 = (int)fminf(fmaxf(x0f, -2.f), (float)W);
    t.y0 = (int)fminf(fmaxf(y0f, -2.f), (float)H);
    t.z0 = (int)fminf(fmaxf(z0f, -2.f), (float)D);
    return t;
}

// utils.index_point_feature (utils.py:357-383): trilinear, zeros padding, align_corners=True.
// All sixteen 16-byte loads are issued unconditionally (indices clamped, out-of-volume corners get
// weight 0) so they are in flight together instead of one DRAM latency per corner.
// VT = __half: sc.vol points at an fp16 [D,Hp,Wp,8] image, one 16-byte load per corner (eight in flight); every value
// is widened exactly (__half2float) and enters the same FMAs in the same order, so the result is bit-identical to the
// fp32 path on the volume `vol.half().float()`.
template <typename VT = float>
__device__ __forceinline__ void sample_volume(const SceneDev& sc, float nx, float ny, float nz, float* out8) {
    const int W = sc.Wp, H = sc.Hp, D = sc.D;
    Trilinear t = trilinear_corners(sc, nx, ny, nz);
    int xo[2], yo[2], zo[2];
#pragma unroll
    for (int d = 0; d < 2; ++d) {
        const int x = t.x0 + d, y = t.y0 + d, z = t.z0 + d;
        if ((unsigned)x >= (unsigned)W) t.wx[d] = 0.f;     // zeros padding: the tap contributes nothing
        if ((unsigned)y >= (unsigned)H) t.wy[d] = 0.f;
        if ((unsigned)z >= (unsigned)D) t.wz[d] = 0.f;
        xo[d] = min(max(x, 0), W - 1); yo[d] = min(max(y, 0), H - 1); zo[d] = min(max(z, 0), D - 1);
    }
    float4 va[8], vb[8];
    if constexpr (std::is_same<VT, __half>::value) {
        uint4 hv[8];
#pragma unroll
        for (int c = 0; c < 8; ++c)
            hv[c] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(sc.vol) +
                                                         (((size_t)zo[c >> 2] * H + yo[(c >> 1) & 1]) * W + xo[c & 1]) * 8));
        auto lo = [](uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u & 0xffffu))); };
        auto hi = [](uint32_t u) { return __half2float(__ushort_as_half((unsigned short)(u >> 16))); };
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            va[c] = make_float4(lo(hv[c].x), hi(hv[c].x), lo(hv[c].y), hi(hv[c].y));
            vb[c] = make_float4(lo(hv[c].z), hi(hv[c].z), lo(hv[c].w), hi(hv[c].w));
        }
    } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const float4* p = reinterpret_cast<const float4*>(
                sc.vol + (((size_t)zo[c >> 2] * H + yo[(c >> 1) & 1]) * W + xo[c & 1]) * 8);
            va[c] = __ldg(p); vb[c] = __ldg(p + 1);
        }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) out8[c] = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {                          // accumulation order as aten: x fastest, then y, then z
        const float wgt = t.wx[c & 1] * t.wy[(c >> 1) & 1] * t.wz[c >> 2];
        out8[0] = fmaf(va[c].x, wgt, out8[0]); out8[1] = fmaf(va[c].y, wgt, out8[1]);
        out8[2] = fmaf(va[c].z, wgt, out8[2]); out8[3] = fmaf(va[c].w, wgt, out8[3]);
        out8[4] = fmaf(vb[c].x, wgt, out8[4]); out8[5] = fmaf(vb[c].y, wgt, out8[5]);
        out8[6] = fmaf(vb[c].z, wgt, out8[6]); out8[7] = fmaf(vb[c].w, wgt, out8[7]);
    }
}

// utils.build_color_volume (utils.py:300-332): bilinear, BORDER padding, strict in-bounds mask.
// out4 = (r, g, b, mask)
template <bool PRECISE = true>
__device__ __forceinline__ void sample_color(const SceneDev& sc, const Cams& cams, int v, float px, float py, float pz, float* out4) {
    const int W = sc.W, H = sc.H;
    float u, vv, zc;
    project_view<PRECISE>(cams.w2c[v], cams.K[v], px, py, pz, (float)(W - 1), (float)(H - 1), u, vv, zc);
    float gx = u * 2.f - 1.f, gy = vv * 2.f - 1.f;
    float ix = ((gx + 1.f) * 0.5f) * (float)(W - 1);
    float iy = ((gy + 1.f) * 0.5f) * (float)(H - 1);
    ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));    // border: clip the source index
    iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
    float x0f = floorf(ix), y0f = floorf(iy);
    float wx1 = ix - x0f, wy1 = iy - y0f, wx0 = (x0f + 1.f) - ix, wy0 = (y0f + 1.f) - iy;
    int x0 = (int)x0f, y0 = (int)y0f;
    if (!(ix == ix)) { x0 = 0; }   // NaN coordinate: keep addresses legal; weights propagate NaN
    if (!(iy == iy)) { y0 = 0; }
    int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);   // the clipped tap always has weight 0
    const float4* img = sc.imgs + (size_t)v * H * W;
    float4 nw = __ldg(img + (size_t)y0 * W + x0), ne = __ldg(img + (size_t)y0 * W + x1);
    float4 sw = __ldg(img + (size_t)y1 * W + x0), se = __ldg(img + (size_t)y1 * W + x1);
    float a = wx0 * wy0, b = wx1 * wy0, c = wx0 * wy1, d = wx1 * wy1;
    out4[0] = fmaf(se.x, d, fmaf(sw.x, c, fmaf(ne.x, b, nw.x * a)));
    out4[1] = fmaf(se.y, d, fmaf(sw.y, c, fmaf(ne.y, b, nw.y * a)));
    out4[2] = fmaf(se.z, d, fmaf(sw.z, c, fmaf(ne.z, b, nw.z * a)));
    out4[3] = (gx > -1.f && gx < 1.f && gy > -1.f && gy < 1.f) ? 1.f : 0.f;
}

// gen_dir_feature (renderer.py:111-122,142-147): unit direction in the reference camera frame
template <bool PRECISE = true>
__device__ __forceinline__ void view_dir(const Cams& cams, float dx, float dy, float dz, float* out3) {
    if (PRECISE) {
        float n = sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
        dx = __fdiv_rn(dx, n); dy = __fdiv_rn(dy, n); dz = __fdiv_rn(dz, n);
    } else {
        const float rn = rsqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
        dx *= rn; dy *= rn; dz *= rn;
    }
    const float* R = cams.w2c[0];
    out3[0] = fmaf(dz, R[2], fmaf(dy, R[1], dx * R[0]));
    out3[1] = fmaf(dz, R[6], fmaf(dy, R[5], dx * R[4]));
    out3[2] = fmaf(dz, R[10], fmaf(dy, R[9], dx * R[8]));
}

}  // namespace mvsn
