// C-ABI entry points (include/mvsnerf_b200.h): argument checking, layout helpers, weight
// packing and the render dispatch.  Kernels live in the sibling .cu files.
#include "render_frontend.cuh"

namespace mvsn {

// ------------------------------------------------------------------------------------------
// error channel
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 148;
    static int cache[64] = {0};
    if (dev < 64 && cache[dev]) return cache[dev];
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
    if (dev < 64) cache[dev] = n;
    return n;
}

// ------------------------------------------------------------------------------------------
// layout kernels
// ------------------------------------------------------------------------------------------
__global__ void pack_images_kernel(const float* __restrict__ src, float4* __restrict__ dst, int V, int HW) {
    const long long n = (long long)V * HW;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(i / HW), p = (int)(i - (long long)v * HW);
        const float* s = src + (size_t)v * 3 * HW + p;
        dst[i] = make_float4(s[0], s[HW], s[2 * (size_t)HW], 0.f);
    }
}

// [8][nvox] <-> [nvox][8]
__global__ void vol_to_cl_kernel(const float* __restrict__ src, float4* __restrict__ dst, long long nvox) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox; i += (long long)gridDim.x * blockDim.x) {
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] = __ldg(src + c * nvox + i);
        dst[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
        dst[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
    }
}
__global__ void vol_from_cl_kernel(const float4* __restrict__ src, float* __restrict__ dst, long long nvox) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox; i += (long long)gridDim.x * blockDim.x) {
        float4 a = __ldg(src + 2 * i), b = __ldg(src + 2 * i + 1);
        dst[0 * nvox + i] = a.x; dst[1 * nvox + i] = a.y; dst[2 * nvox + i] = a.z; dst[3 * nvox + i] = a.w;
        dst[4 * nvox + i] = b.x; dst[5 * nvox + i] = b.y; dst[6 * nvox + i] = b.z; dst[7 * nvox + i] = b.w;
    }
}

// rays [n][8] = (origin, direction, near, far) of one camera: d = directions @ c2w[:3,:3]^T, o = c2w[:3,3]
// (data/ray_utils.py:32-53 get_rays + the notebooks' cat with near / far)
__global__ void make_rays_kernel(const float* __restrict__ dirs, const float* __restrict__ c2w, float near, float far, int n,
                                 float4* __restrict__ rays) {
    __shared__ float m[12];
    if (threadIdx.x < 12) m[threadIdx.x] = __ldg(c2w + threadIdx.x);           // rows of [R | t], row-major [.,4]
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float x = __ldg(dirs + 3 * (size_t)i), y = __ldg(dirs + 3 * (size_t)i + 1), z = __ldg(dirs + 3 * (size_t)i + 2);
        const float dx = fmaf(z, m[2], fmaf(y, m[1], x * m[0]));
        const float dy = fmaf(z, m[6], fmaf(y, m[5], x * m[4]));
        const float dz = fmaf(z, m[10], fmaf(y, m[9], x * m[8]));
        rays[2 * (size_t)i] = make_float4(m[3], m[7], m[11], dx);
        rays[2 * (size_t)i + 1] = make_float4(dy, dz, near, far);
    }
}

// ------------------------------------------------------------------------------------------
// fp32 MLP weight image
// ------------------------------------------------------------------------------------------
struct MlpPtrs { const float* p[MVSN_N_MLP_TENSORS]; };
// indices into the 22-tensor array (see header)
enum { I_W0 = 0, I_B0 = 1, I_WB = 12, I_BB = 13, I_WV = 14, I_BV = 15, I_WF = 16, I_BF = 17,
       I_WA = 18, I_BA = 19, I_WR = 20, I_BR = 21 };

// dst[k][n] (ld = ldn) = src[n][src_col0 + k] for k < kreal, 0 for kreal <= k < kpad
__device__ void transpose_into(float* dst, int ldn, int nout, int kpad, const float* src, int src_ld,
                               int src_col0, int kreal, int tid, int nthreads) {
    for (int i = tid; i < kpad * nout; i += nthreads) {
        const int k = i / nout, n = i - k * nout;
        dst[k * ldn + n] = k < kreal ? src[(size_t)n * src_ld + src_col0 + k] : 0.f;
    }
}
__device__ void copy_into(float* dst, const float* src, int n, int npad, int tid, int nthreads) {
    for (int i = tid; i < npad; i += nthreads) dst[i] = i < n ? src[i] : 0.f;
}

__global__ void pack_mlp_fp32_kernel(MlpPtrs w, float* __restrict__ out) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    using namespace w32;
    transpose_into(out + WB, 128, 128, 32, w.p[I_WB], 20, 0, 20, tid, nt);
    copy_into(out + BB, w.p[I_BB], 128, 128, tid, nt);
    transpose_into(out + W0, 128, 128, 64, w.p[I_W0], 63, 0, 63, tid, nt);
    copy_into(out + B0, w.p[I_B0], 128, 128, tid, nt);
    for (int l = 1; l <= 4; ++l) {
        transpose_into(out + W1 + (l - 1) * LSTR, 128, 128, 128, w.p[2 * l], 128, 0, 128, tid, nt);
        copy_into(out + W1 + (l - 1) * LSTR + 128 * 128, w.p[2 * l + 1], 128, 128, tid, nt);
    }
    transpose_into(out + W5, 128, 128, 64, w.p[10], 191, 0, 63, tid, nt);             // pe part
    transpose_into(out + W5 + 64 * 128, 128, 128, 128, w.p[10], 191, 63, 128, tid, nt); // h part
    copy_into(out + B5, w.p[11], 128, 128, tid, nt);
    copy_into(out + WA, w.p[I_WA], 128, 128, tid, nt);
    copy_into(out + BA, w.p[I_BA], 1, 4, tid, nt);
    transpose_into(out + WF, 128, 128, 128, w.p[I_WF], 128, 0, 128, tid, nt);
    copy_into(out + BF, w.p[I_BF], 128, 128, tid, nt);
    transpose_into(out + WV, 64, 64, 128, w.p[I_WV], 131, 0, 128, tid, nt);
    transpose_into(out + WVD, 64, 64, 4, w.p[I_WV], 131, 128, 3, tid, nt);
    copy_into(out + BV, w.p[I_BV], 64, 64, tid, nt);
    // rgb_linear [3][64] is used row-wise (dot products), no transpose
    for (int i = tid; i < 4 * 64; i += nt) out[WR + i] = i < 3 * 64 ? w.p[I_WR][i] : 0.f;
    copy_into(out + BR, w.p[I_BR], 3, 4, tid, nt);
}

static int make_scene(const mvsn_render_scene* s, SceneDev& d) {
    MVSN_REQUIRE(s != nullptr, MVSN_ENULL, "scene is NULL");
    MVSN_REQUIRE(s->volume_dhwc && s->imgs_hwc4 && s->mlp_packed, MVSN_ENULL, "scene has a NULL buffer");
    MVSN_REQUIRE(s->V == 3, MVSN_EBADSHAPE, "V=%d: the v0 MLP takes 8 + 4*3 feature channels", s->V);
    MVSN_REQUIRE(s->D > 0 && s->Hp > 0 && s->Wp > 0 && s->H > 1 && s->W > 1, MVSN_EBADSHAPE, "bad scene dims");
    MVSN_REQUIRE(aligned16(s->volume_dhwc) && aligned16(s->imgs_hwc4) && aligned16(s->mlp_packed), MVSN_EALIGN,
                 "scene buffers must be 16-byte aligned");
    d.vol = s->volume_dhwc; d.imgs = reinterpret_cast<const float4*>(s->imgs_hwc4);
    d.D = s->D; d.Hp = s->Hp; d.Wp = s->Wp; d.V = s->V; d.H = s->H; d.W = s->W;
    MVSN_REQUIRE(s->w2cs && s->intrinsics, MVSN_ENULL, "scene camera pointers are NULL");
    d.w2cs = s->w2cs; d.intrinsics = s->intrinsics;
    d.white_bkgd = s->white_bkgd;
    return MVSN_OK;
}

// scene->mlp_mode without / with the MVSN_VOLUME_F16 flag
static int mlp_mode_of(const mvsn_render_scene* scene) { return scene->mlp_mode & ~MVSN_VOLUME_F16; }
static bool half_volume(const mvsn_render_scene* scene) { return (scene->mlp_mode & MVSN_VOLUME_F16) != 0; }

static int dispatch_render(const mvsn_render_scene* scene, const SceneDev& sc, const RenderIO& io, bool fast,
                           cudaStream_t stream) {
    const bool hv = half_volume(scene);
    switch (mlp_mode_of(scene)) {
        case MVSN_MLP_FP32:
            MVSN_REQUIRE(!hv, MVSN_EUNSUPPORTED, "MVSN_MLP_FP32 reads an fp32 volume only (MVSN_VOLUME_F16 given)");
            return launch_render_fp32(sc, io, fast, static_cast<const float*>(scene->mlp_packed), stream);
        case MVSN_MLP_TC_HALF:
        case MVSN_MLP_TC_PAIR:
            return launch_render_wg(sc, io, fast, false, scene->mlp_packed, stream, nullptr, nullptr, hv);
        case MVSN_MLP_TC_SPLIT:
            return launch_render_wg(sc, io, fast, true, scene->mlp_packed, stream, nullptr, nullptr, hv);
        default:
            set_error("mlp_mode %d is not available in this build", scene->mlp_mode);
            return MVSN_EUNSUPPORTED;
    }
}

}  // namespace mvsn

using namespace mvsn;

extern "C" {

const char* mvsn_last_error(void) { return g_err; }
int mvsn_abi_version(void) { return 2; }

size_t mvsn_mlp_packed_bytes(int mode) {
    switch (mode & ~MVSN_VOLUME_F16) {
        case MVSN_MLP_FP32: return (size_t)w32::TOTAL * sizeof(float);
        case MVSN_MLP_TC_HALF:
        case MVSN_MLP_TC_PAIR: return mlp_wg_packed_bytes(false);
        case MVSN_MLP_TC_SPLIT: return mlp_wg_packed_bytes(true);
        default: return 0;
    }
}

int mvsn_mlp_pack(const float* const* w, int mode, void* packed, size_t packed_bytes, void* stream) {
    MVSN_RANGE("mvsn_mlp_pack");
    mode &= ~MVSN_VOLUME_F16;                             // the weight image does not depend on the volume's storage
    MVSN_REQUIRE(w && packed, MVSN_ENULL, "mvsn_mlp_pack: NULL argument");
    const size_t need = mvsn_mlp_packed_bytes(mode);
    MVSN_REQUIRE(need != 0, MVSN_EUNSUPPORTED, "mvsn_mlp_pack: mode %d not available", mode);
    MVSN_REQUIRE(packed_bytes >= need, MVSN_EWORKSPACE, "mvsn_mlp_pack: need %zu bytes, got %zu", need, packed_bytes);
    MVSN_REQUIRE(aligned16(packed), MVSN_EALIGN, "mvsn_mlp_pack: packed buffer must be 16-byte aligned");
    MlpPtrs p;
    for (int i = 0; i < MVSN_N_MLP_TENSORS; ++i) {
        MVSN_REQUIRE(w[i] != nullptr, MVSN_ENULL, "mvsn_mlp_pack: tensor %d is NULL", i);
        p.p[i] = w[i];
    }
    if (mode == MVSN_MLP_TC_HALF || mode == MVSN_MLP_TC_PAIR) return pack_mlp_wg(w, false, packed, (cudaStream_t)stream);
    if (mode == MVSN_MLP_TC_SPLIT) return pack_mlp_wg(w, true, packed, (cudaStream_t)stream);
    pack_mlp_fp32_kernel<<<64, 256, 0, (cudaStream_t)stream>>>(p, static_cast<float*>(packed));
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

int mvsn_pack_images(const float* imgs, int V, int H, int W, float* out, void* stream) {
    MVSN_REQUIRE(imgs && out, MVSN_ENULL, "mvsn_pack_images: NULL argument");
    MVSN_REQUIRE(V > 0 && H > 0 && W > 0, MVSN_EBADSHAPE, "mvsn_pack_images: bad shape");
    MVSN_REQUIRE(aligned16(out), MVSN_EALIGN, "mvsn_pack_images: output must be 16-byte aligned");
    const long long n = (long long)V * H * W;
    pack_images_kernel<<<cdiv(n, 256) < 4096 ? cdiv(n, 256) : 4096, 256, 0, (cudaStream_t)stream>>>(
        imgs, reinterpret_cast<float4*>(out), V, H * W);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

int mvsn_volume_to_channels_last(const float* src, int D, int Hp, int Wp, float* dst, void* stream) {
    MVSN_REQUIRE(src && dst, MVSN_ENULL, "mvsn_volume_to_channels_last: NULL argument");
    MVSN_REQUIRE(aligned16(dst), MVSN_EALIGN, "mvsn_volume_to_channels_last: output must be 16-byte aligned");
    const long long n = (long long)D * Hp * Wp;
    MVSN_REQUIRE(n > 0, MVSN_EBADSHAPE, "mvsn_volume_to_channels_last: bad shape");
    vol_to_cl_kernel<<<cdiv(n, 256) < 8192 ? cdiv(n, 256) : 8192, 256, 0, (cudaStream_t)stream>>>(
        src, reinterpret_cast<float4*>(dst), n);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

int mvsn_volume_from_channels_last(const float* src, int D, int Hp, int Wp, float* dst, void* stream) {
    MVSN_REQUIRE(src && dst, MVSN_ENULL, "mvsn_volume_from_channels_last: NULL argument");
    MVSN_REQUIRE(aligned16(src), MVSN_EALIGN, "mvsn_volume_from_channels_last: input must be 16-byte aligned");
    const long long n = (long long)D * Hp * Wp;
    MVSN_REQUIRE(n > 0, MVSN_EBADSHAPE, "mvsn_volume_from_channels_last: bad shape");
    vol_from_cl_kernel<<<cdiv(n, 256) < 8192 ? cdiv(n, 256) : 8192, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(src), dst, n);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

int mvsn_volume_to_half(const void* src, int src_half, int src_planar, int D, int Hp, int Wp, void* vol_dhwc_f16,
                        void* stream) {
    MVSN_RANGE("mvsn_volume_to_half");
    MVSN_REQUIRE(src && vol_dhwc_f16, MVSN_ENULL, "mvsn_volume_to_half: NULL argument");
    MVSN_REQUIRE(D > 0 && Hp > 0 && Wp > 0, MVSN_EBADSHAPE, "mvsn_volume_to_half: D=%d Hp=%d Wp=%d", D, Hp, Wp);
    MVSN_REQUIRE(aligned16(vol_dhwc_f16), MVSN_EALIGN, "mvsn_volume_to_half: output must be 16-byte aligned");
    MVSN_REQUIRE(reinterpret_cast<uintptr_t>(src) % (src_half ? 2 : 4) == 0, MVSN_EALIGN,
                 "mvsn_volume_to_half: input not aligned to its element size");
    const long long n = (long long)D * Hp * Wp;
    return launch_volume_to_half(src, src_half != 0, src_planar != 0, n, vol_dhwc_f16, (cudaStream_t)stream);
}

int mvsn_render_samples(const mvsn_render_scene* scene, const float* rays_pts, const float* rays_ndc,
                        const float* z_vals, const float* rays_dir, int N, int S, float* rgb, float* depth,
                        float* weights, float* alpha, float* input_feat, void* stream) {
    MVSN_RANGE("mvsn_render_samples");
    SceneDev sc;
    int rc = make_scene(scene, sc);
    if (rc) return rc;
    MVSN_REQUIRE(N >= 0 && S > 0, MVSN_EBADSHAPE, "mvsn_render_samples: N=%d S=%d", N, S);
    if (N == 0) return MVSN_OK;
    MVSN_REQUIRE(rays_pts && rays_ndc && z_vals && rays_dir && rgb && depth, MVSN_ENULL,
                 "mvsn_render_samples: NULL required pointer");
    MVSN_REQUIRE(!input_feat || aligned16(input_feat), MVSN_EALIGN, "input_feat must be 16-byte aligned");
    RenderIO io{};
    io.pts = rays_pts; io.ndc = rays_ndc; io.z = z_vals; io.dirs = rays_dir;
    io.N = N; io.S = S;
    io.rgb = rgb; io.depth = depth; io.weights = weights; io.alpha = alpha; io.input_feat = input_feat;
    return dispatch_render(scene, sc, io, false, (cudaStream_t)stream);
}

int mvsn_render_samples_stop(const mvsn_render_scene* scene, const float* rays_pts, const float* rays_ndc,
                             const float* z_vals, const float* rays_dir, int N, int S, float t_stop, float* rgb,
                             float* depth, unsigned long long* tiles_done, void* stream) {
    MVSN_RANGE("mvsn_render_samples_stop");
    const char* what = "mvsn_render_samples_stop";
    SceneDev sc;
    int rc = make_scene(scene, sc);
    if (rc) return rc;
    MVSN_REQUIRE(N >= 0 && S > 0, MVSN_EBADSHAPE, "%s: N=%d S=%d", what, N, S);
    MVSN_REQUIRE(rays_pts && rays_ndc && z_vals && rays_dir && rgb && depth, MVSN_ENULL, "%s: NULL required pointer", what);
    MVSN_REQUIRE(t_stop >= 0.f, MVSN_EBADSHAPE, "%s: t_stop=%g must be >= 0 (not NaN)", what, (double)t_stop);
    const int mode = mlp_mode_of(scene);
    MVSN_REQUIRE(mode == MVSN_MLP_TC_HALF || mode == MVSN_MLP_TC_PAIR || mode == MVSN_MLP_TC_SPLIT,
                 MVSN_EUNSUPPORTED, "%s: mlp_mode %d has no early ray termination (tensor-core modes only)", what,
                 scene->mlp_mode);
    MVSN_REQUIRE(reinterpret_cast<uintptr_t>(tiles_done) % 8 == 0, MVSN_EALIGN, "%s: tiles_done must be 8-byte aligned", what);
    if (N == 0) return MVSN_OK;
    RenderIO io{};
    io.pts = rays_pts; io.ndc = rays_ndc; io.z = z_vals; io.dirs = rays_dir;
    io.N = N; io.S = S;
    io.rgb = rgb; io.depth = depth;
    return launch_render_wg(sc, io, false, mode == MVSN_MLP_TC_SPLIT, scene->mlp_packed, (cudaStream_t)stream, &t_stop,
                            tiles_done, half_volume(scene), nullptr, nullptr);
}

// host-side scalars of the in-kernel ray march exactly as utils.get_ndc_coordinate forms them (python floats -> fp32)
static RayGenDev make_ray_gen(const mvsn_render_scene* scene, const mvsn_ray_params* rp) {
    RayGenDev rg;
    rg.near = rp->ndc_near;
    rg.far_minus_near = (float)((double)rp->ndc_far - (double)rp->ndc_near);
    rg.inv_near = (float)(1.0 / (double)rp->ndc_near);
    rg.inv_far_minus_inv_near = (float)(1.0 / (double)rp->ndc_far - 1.0 / (double)rp->ndc_near);
    rg.pad = rp->pad;
    rg.wf = (float)scene->W / 4.0f;     // (inv_scale + 1) / 4, utils.py:139
    rg.hf = (float)scene->H / 4.0f;
    rg.lindisp = rp->lindisp;
    return rg;
}

static int render_rays_impl(const mvsn_render_scene* scene, const mvsn_ray_params* rp, const float* rays,
                            const float* t_steps, int N, int S, float* rgb, float* depth, float* weights,
                            float* alpha, float* input_feat, const mvsn_peer_sink* sink, void* stream) {
    MVSN_RANGE("mvsn_render_rays");
    SceneDev sc;
    int rc = make_scene(scene, sc);
    if (rc) return rc;
    MVSN_REQUIRE(rp != nullptr, MVSN_ENULL, "mvsn_render_rays: ray params NULL");
    MVSN_REQUIRE(N >= 0 && S > 0, MVSN_EBADSHAPE, "mvsn_render_rays: N=%d S=%d", N, S);
    if (N == 0) return MVSN_OK;
    MVSN_REQUIRE(rays && t_steps && (sink || (rgb && depth)), MVSN_ENULL, "mvsn_render_rays: NULL required pointer");
    MVSN_REQUIRE(aligned16(rays), MVSN_EALIGN, "rays must be 16-byte aligned");
    MVSN_REQUIRE(!input_feat || aligned16(input_feat), MVSN_EALIGN, "input_feat must be 16-byte aligned");
    RenderIO io{};
    io.rays = rays; io.t_steps = t_steps;
    io.N = N; io.S = S;
    io.rgb = rgb; io.depth = depth; io.weights = weights; io.alpha = alpha; io.input_feat = input_feat;
    io.rg = make_ray_gen(scene, rp);
    if (sink) {
        MVSN_REQUIRE(sink->n_peers >= 1 && sink->n_peers <= MVSN_MAX_PEERS, MVSN_EBADSHAPE,
                     "peer sink: n_peers=%d (1..%d)", sink->n_peers, MVSN_MAX_PEERS);
        MVSN_REQUIRE(sink->first_pixel >= 0, MVSN_EBADSHAPE, "peer sink: first_pixel < 0");
        for (int p = 0; p < sink->n_peers; ++p) {
            MVSN_REQUIRE(sink->frame[p] != nullptr, MVSN_ENULL, "peer sink: frame[%d] is NULL", p);
            MVSN_REQUIRE(aligned16(sink->frame[p]), MVSN_EALIGN, "peer sink: frame[%d] must be 16-byte aligned", p);
            io.sink[p] = reinterpret_cast<float4*>(sink->frame[p]);
        }
        io.n_sink = sink->n_peers;
        io.sink_first = sink->first_pixel;
    }
    return dispatch_render(scene, sc, io, true, (cudaStream_t)stream);
}

int mvsn_render_rays(const mvsn_render_scene* scene, const mvsn_ray_params* rp, const float* rays,
                     const float* t_steps, int N, int S, float* rgb, float* depth, float* weights,
                     float* alpha, float* input_feat, void* stream) {
    return render_rays_impl(scene, rp, rays, t_steps, N, S, rgb, depth, weights, alpha, input_feat, nullptr, stream);
}

// mvsn_render_rays_stop and, with `occ`, mvsn_render_rays_occ (`what`: the entry's name for messages)
static int render_rays_stop_entry(const char* what, const mvsn_render_scene* scene, const mvsn_ray_params* rp,
                                  const float* rays, const float* t_steps, int N, int S, float t_stop,
                                  const mvsn_occupancy* occ, float* rgb, float* depth, unsigned long long* tiles_done,
                                  void* workspace, size_t workspace_bytes, void* stream) {
    SceneDev sc;
    int rc = make_scene(scene, sc);
    if (rc) return rc;
    MVSN_REQUIRE(rp != nullptr, MVSN_ENULL, "%s: ray params NULL", what);
    MVSN_REQUIRE(N >= 0 && S > 0, MVSN_EBADSHAPE, "%s: N=%d S=%d", what, N, S);
    MVSN_REQUIRE(rays && t_steps && rgb && depth, MVSN_ENULL, "%s: NULL required pointer", what);
    MVSN_REQUIRE(t_stop >= 0.f, MVSN_EBADSHAPE, "%s: t_stop=%g must be >= 0 (not NaN)", what, (double)t_stop);
    const int mode = mlp_mode_of(scene);
    MVSN_REQUIRE(mode == MVSN_MLP_TC_HALF || mode == MVSN_MLP_TC_PAIR || mode == MVSN_MLP_TC_SPLIT,
                 MVSN_EUNSUPPORTED, "%s: mlp_mode %d has no early ray termination (tensor-core modes only)", what,
                 scene->mlp_mode);
    MVSN_REQUIRE(aligned16(rays), MVSN_EALIGN, "rays must be 16-byte aligned");
    MVSN_REQUIRE(reinterpret_cast<uintptr_t>(tiles_done) % 8 == 0, MVSN_EALIGN, "%s: tiles_done must be 8-byte aligned", what);
    if (occ) {
        MVSN_REQUIRE(occ->bits != nullptr, MVSN_ENULL, "%s: occupancy->bits is NULL", what);
        MVSN_REQUIRE(reinterpret_cast<uintptr_t>(occ->bits) % 4 == 0, MVSN_EALIGN, "%s: occupancy->bits must be 4-byte aligned",
                     what);
        MVSN_REQUIRE(occ->D == scene->D && occ->Hp == scene->Hp && occ->Wp == scene->Wp && occ->D >= 2 && occ->Hp >= 2 &&
                     occ->Wp >= 2, MVSN_EBADSHAPE, "%s: occupancy grid %dx%dx%d does not match the scene's volume %dx%dx%d",
                     what, occ->D, occ->Hp, occ->Wp, scene->D, scene->Hp, scene->Wp);
        MVSN_REQUIRE(workspace != nullptr, MVSN_ENULL, "%s: workspace is NULL", what);
        MVSN_REQUIRE(aligned16(workspace), MVSN_EALIGN, "%s: workspace must be 16-byte aligned", what);
        MVSN_REQUIRE(workspace_bytes >= occupancy_ranges_bytes(N), MVSN_EWORKSPACE, "%s: workspace needs %zu bytes, got %zu",
                     what, occupancy_ranges_bytes(N), workspace_bytes);
    }
    if (N == 0) return MVSN_OK;
    RenderIO io{};
    io.rays = rays; io.t_steps = t_steps;
    io.N = N; io.S = S;
    io.rgb = rgb; io.depth = depth;
    io.rg = make_ray_gen(scene, rp);
    return launch_render_wg(sc, io, true, mode == MVSN_MLP_TC_SPLIT, scene->mlp_packed, (cudaStream_t)stream,
                            &t_stop, tiles_done, half_volume(scene), occ ? occ->bits : nullptr,
                            occ ? static_cast<int2*>(workspace) : nullptr);
}

int mvsn_render_rays_stop(const mvsn_render_scene* scene, const mvsn_ray_params* rp, const float* rays,
                          const float* t_steps, int N, int S, float t_stop, float* rgb, float* depth,
                          unsigned long long* tiles_done, void* stream) {
    MVSN_RANGE("mvsn_render_rays_stop");
    return render_rays_stop_entry("mvsn_render_rays_stop", scene, rp, rays, t_steps, N, S, t_stop, nullptr, rgb, depth,
                                  tiles_done, nullptr, 0, stream);
}

size_t mvsn_render_rays_occ_workspace_bytes(int N, int S) {
    return N >= 0 && S > 0 ? occupancy_ranges_bytes(N) : 0;
}

int mvsn_render_rays_occ(const mvsn_render_scene* scene, const mvsn_ray_params* rp, const float* rays,
                         const float* t_steps, int N, int S, float t_stop, const mvsn_occupancy* occupancy, float* rgb,
                         float* depth, unsigned long long* tiles_done, void* workspace, size_t workspace_bytes,
                         void* stream) {
    MVSN_RANGE("mvsn_render_rays_occ");
    MVSN_REQUIRE(occupancy != nullptr, MVSN_ENULL, "mvsn_render_rays_occ: occupancy is NULL");
    return render_rays_stop_entry("mvsn_render_rays_occ", scene, rp, rays, t_steps, N, S, t_stop, occupancy, rgb, depth,
                                  tiles_done, workspace, workspace_bytes, stream);
}

size_t mvsn_occupancy_bytes(int D, int Hp, int Wp) {
    return D > 0 && Hp > 0 && Wp > 0 ? occupancy_words(D, Hp, Wp) * 4 : 0;
}

size_t mvsn_build_occupancy_workspace_bytes(int D, int Hp, int Wp) { return occupancy_workspace_bytes(D, Hp, Wp); }

int mvsn_build_occupancy(const mvsn_render_scene* scene, const mvsn_ray_params* rp, int dilate, uint32_t* bits,
                         void* workspace, size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_build_occupancy");
    SceneDev sc;
    int rc = make_scene(scene, sc);
    if (rc) return rc;
    MVSN_REQUIRE(rp && bits && workspace, MVSN_ENULL, "mvsn_build_occupancy: NULL argument");
    MVSN_REQUIRE(mlp_mode_of(scene) == MVSN_MLP_TC_SPLIT, MVSN_EUNSUPPORTED,
                 "mvsn_build_occupancy: scene->mlp_mode %d (the MVSN_MLP_TC_SPLIT image, optionally | MVSN_VOLUME_F16)",
                 scene->mlp_mode);
    MVSN_REQUIRE(scene->D >= 2 && scene->Hp >= 2 && scene->Wp >= 2, MVSN_EBADSHAPE,
                 "mvsn_build_occupancy: volume %dx%dx%d (every dim >= 2)", scene->D, scene->Hp, scene->Wp);
    MVSN_REQUIRE(dilate >= 0 && dilate <= 8, MVSN_EBADSHAPE, "mvsn_build_occupancy: dilate=%d (0..8)", dilate);
    MVSN_REQUIRE(reinterpret_cast<uintptr_t>(bits) % 4 == 0, MVSN_EALIGN, "mvsn_build_occupancy: bits must be 4-byte aligned");
    MVSN_REQUIRE(aligned16(workspace), MVSN_EALIGN, "mvsn_build_occupancy: workspace must be 16-byte aligned");
    const size_t need = occupancy_workspace_bytes(scene->D, scene->Hp, scene->Wp);
    MVSN_REQUIRE(workspace_bytes >= need, MVSN_EWORKSPACE, "mvsn_build_occupancy: workspace needs %zu bytes, got %zu", need,
                 workspace_bytes);
    return build_occupancy(sc, make_ray_gen(scene, rp), scene->mlp_packed, half_volume(scene), dilate, bits, workspace,
                           (cudaStream_t)stream);
}

size_t mvsn_build_density_workspace_bytes(int D, int Hp, int Wp) { return density_workspace_bytes(D, Hp, Wp); }

int mvsn_build_density(const mvsn_render_scene* scene, const mvsn_ray_params* rp, float* sigma, void* workspace,
                       size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_build_density");
    SceneDev sc;
    int rc = make_scene(scene, sc);
    if (rc) return rc;
    MVSN_REQUIRE(rp && sigma && workspace, MVSN_ENULL, "mvsn_build_density: NULL argument");
    MVSN_REQUIRE(mlp_mode_of(scene) == MVSN_MLP_FP32, MVSN_EUNSUPPORTED,
                 "mvsn_build_density: scene->mlp_mode %d (the MVSN_MLP_FP32 image, optionally | MVSN_VOLUME_F16)",
                 scene->mlp_mode);
    MVSN_REQUIRE(scene->D >= 2 && scene->Hp >= 2 && scene->Wp >= 2, MVSN_EBADSHAPE,
                 "mvsn_build_density: volume %dx%dx%d (every dim >= 2)", scene->D, scene->Hp, scene->Wp);
    MVSN_REQUIRE(reinterpret_cast<uintptr_t>(sigma) % 4 == 0, MVSN_EALIGN, "mvsn_build_density: sigma must be 4-byte aligned");
    MVSN_REQUIRE(aligned16(workspace), MVSN_EALIGN, "mvsn_build_density: workspace must be 16-byte aligned");
    const size_t need = density_workspace_bytes(scene->D, scene->Hp, scene->Wp);
    MVSN_REQUIRE(workspace_bytes >= need, MVSN_EWORKSPACE, "mvsn_build_density: workspace needs %zu bytes, got %zu", need,
                 workspace_bytes);
    return build_density(sc, make_ray_gen(scene, rp), static_cast<const float*>(scene->mlp_packed), half_volume(scene),
                         sigma, workspace, (cudaStream_t)stream);
}

int mvsn_sample_importance(const mvsn_render_scene* scene, const mvsn_ray_params* rp, const mvsn_density* density,
                           const float* rays, const float* t_steps, const float* jitter, const float* z_vals,
                           const float* ndc, const float* u, int N, int S, int K, float* z_out, float* pts_out,
                           float* ndc_out, void* stream) {
    MVSN_RANGE("mvsn_sample_importance");
    const char* what = "mvsn_sample_importance";
    MVSN_REQUIRE(N >= 0 && S >= 3 && K >= 1, MVSN_EBADSHAPE, "%s: N=%d S=%d K=%d (S >= 3, K >= 1)", what, N, S, K);
    MVSN_REQUIRE(S + K <= MAX_IMPORTANCE_SAMPLES, MVSN_EUNSUPPORTED, "%s: S + K = %d (at most %d)", what, S + K,
                 MAX_IMPORTANCE_SAMPLES);
    MVSN_REQUIRE(density && density->sigma && rays && z_out && pts_out, MVSN_ENULL, "%s: NULL required pointer", what);
    MVSN_REQUIRE((t_steps != nullptr) != (z_vals != nullptr), MVSN_ENULL,
                 "%s: exactly one coarse source: t_steps (marched) or z_vals + ndc", what);
    MVSN_REQUIRE(t_steps || ndc, MVSN_ENULL, "%s: z_vals needs ndc", what);
    MVSN_REQUIRE(!z_vals || !jitter, MVSN_EUNSUPPORTED, "%s: jitter applies to the marched source only", what);
    const bool cams = t_steps != nullptr || ndc_out != nullptr;
    MVSN_REQUIRE(!cams || (scene && rp), MVSN_ENULL, "%s: the march and ndc_out need scene and rp", what);
    SceneDev sc{};
    if (scene) {
        int rc = make_scene(scene, sc);
        if (rc) return rc;
    }
    MVSN_REQUIRE(aligned16(rays), MVSN_EALIGN, "%s: rays must be 16-byte aligned", what);
    MVSN_REQUIRE(reinterpret_cast<uintptr_t>(density->sigma) % 4 == 0, MVSN_EALIGN, "%s: density->sigma must be 4-byte aligned",
                 what);
    MVSN_REQUIRE(density->D >= 2 && density->Hp >= 2 && density->Wp >= 2, MVSN_EBADSHAPE,
                 "%s: density grid %dx%dx%d (every dim >= 2)", what, density->D, density->Hp, density->Wp);
    MVSN_REQUIRE(!scene || (density->D == scene->D && density->Hp == scene->Hp && density->Wp == scene->Wp), MVSN_EBADSHAPE,
                 "%s: density grid %dx%dx%d does not match the scene's volume %dx%dx%d", what, density->D, density->Hp,
                 density->Wp, scene ? scene->D : 0, scene ? scene->Hp : 0, scene ? scene->Wp : 0);
    if (N == 0) return MVSN_OK;
    sc.D = density->D; sc.Hp = density->Hp; sc.Wp = density->Wp;
    ImportanceIO io{};
    io.rays = rays; io.t_steps = t_steps; io.jitter = jitter; io.z_in = z_vals; io.ndc_in = ndc;
    io.sigma = density->sigma; io.u = u;
    io.N = N; io.S = S; io.K = K; io.cams = cams;
    io.z_out = z_out; io.pts_out = pts_out; io.ndc_out = ndc_out;
    const RayGenDev rg = cams ? make_ray_gen(scene, rp) : RayGenDev{};
    return launch_importance(sc, rg, io, (cudaStream_t)stream);
}

int mvsn_render_rays_to_peers(const mvsn_render_scene* scene, const mvsn_ray_params* rp, const float* rays,
                              const float* t_steps, int N, int S, const mvsn_peer_sink* sink, float* rgb,
                              float* depth, void* stream) {
    MVSN_REQUIRE(sink != nullptr, MVSN_ENULL, "mvsn_render_rays_to_peers: sink is NULL");
    return render_rays_impl(scene, rp, rays, t_steps, N, S, rgb, depth, nullptr, nullptr, nullptr, sink, stream);
}

int mvsn_make_rays(const float* directions, const float* c2w, float near, float far, int n, float* rays, void* stream) {
    MVSN_RANGE("mvsn_make_rays");
    MVSN_REQUIRE(directions && c2w && rays, MVSN_ENULL, "mvsn_make_rays: NULL argument");
    MVSN_REQUIRE(n >= 0, MVSN_EBADSHAPE, "mvsn_make_rays: n=%d", n);
    MVSN_REQUIRE(aligned16(rays), MVSN_EALIGN, "mvsn_make_rays: rays must be 16-byte aligned");
    if (n == 0) return MVSN_OK;
    make_rays_kernel<<<cdiv(n, 256) < 2048 ? cdiv(n, 256) : 2048, 256, 0, (cudaStream_t)stream>>>(
        directions, c2w, near, far, n, reinterpret_cast<float4*>(rays));
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

// ---- fine-tuning step ------------------------------------------------------------------------------------
// The grad modes of the backward entries: MVSN_GRAD_TC_FULL marches its samples in the kernel, so only the rays
// entries take it.
static bool backward_grad_mode(int grad_mode, bool rays) {
    return grad_mode == MVSN_MLP_FP32 || grad_mode == MVSN_MLP_TC_HALF || (rays && grad_mode == MVSN_GRAD_TC_FULL);
}

static size_t backward_bytes(bool rays, int N, int S, int D, int Hp, int Wp, int grad_mode, bool det, bool stop) {
    return backward_grad_mode(grad_mode, rays) ? backward_layout(N, S, D, Hp, Wp, grad_mode, det, stop).total : 0;
}

// The inputs of a backward entry: the samples (pts, ndc, z, dirs) or, rp set, the rays marched in the kernel.
struct BwdInputs {
    const float *pts, *ndc, *z, *dirs;
    const mvsn_ray_params* rp; const float *rays, *t_steps, *jitter;
};

// Every backward entry, with its checks in the order include/mvsnerf_b200.h states for the fine-tuning entries.
static int backward_entry(const char* what, bool rays, const mvsn_render_scene* scene, const float* const* mlp_w,
                          const BwdInputs& in, int N, int S, int grad_mode, bool det, const BwdStop* stop,
                          const mvsn_render_grads* g, float* const* grad_mlp, float* grad_volume_dhwc, void* workspace,
                          size_t workspace_bytes, void* stream) {
    MVSN_REQUIRE(backward_grad_mode(grad_mode, rays), MVSN_EUNSUPPORTED, "%s: grad_mode %d (%s)", what, grad_mode,
                 rays ? "MVSN_MLP_FP32, MVSN_MLP_TC_HALF or MVSN_GRAD_TC_FULL" : "MVSN_MLP_FP32 or MVSN_MLP_TC_HALF");
    SceneDev sc;
    int rc = make_scene(scene, sc);
    if (rc) return rc;
    MVSN_REQUIRE((!rays || in.rp) && g && mlp_w && grad_mlp, MVSN_ENULL, "%s: NULL argument", what);
    MVSN_REQUIRE(g->rgb || g->target_rgb, MVSN_ENULL, "%s: neither g->rgb nor g->target_rgb given", what);
    for (int i = 0; i < MVSN_N_MLP_TENSORS; ++i)
        MVSN_REQUIRE(mlp_w[i] && grad_mlp[i], MVSN_ENULL, "%s: tensor %d is NULL", what, i);
    if (rays) MVSN_REQUIRE(N == 0 || (in.rays && in.t_steps), MVSN_ENULL, "%s: rays or t_steps is NULL", what);
    else MVSN_REQUIRE(N == 0 || (in.pts && in.ndc && in.z && in.dirs), MVSN_ENULL, "%s: NULL required pointer", what);
    if (stop) {
        MVSN_REQUIRE(stop->t_stop >= 0.f && stop->t_stop <= 1.f, MVSN_EBADSHAPE,
                     "%s: t_stop=%g must be in [0, 1] (not NaN)", what, (double)stop->t_stop);
        MVSN_REQUIRE(!g->weights && !g->alpha && !g->input_feat, MVSN_EUNSUPPORTED,
                     "%s: g->weights / g->alpha / g->input_feat are per-sample cotangents, not defined for dead samples",
                     what);
    }
    MVSN_REQUIRE(aligned16(in.rays), MVSN_EALIGN, "%s: rays must be 16-byte aligned", what);
    MVSN_REQUIRE(!grad_volume_dhwc || aligned16(grad_volume_dhwc), MVSN_EALIGN, "grad_volume_dhwc must be 16-byte aligned");
    if (stop) {
        MVSN_REQUIRE(reinterpret_cast<uintptr_t>(stop->live_samples) % 4 == 0, MVSN_EALIGN,
                     "%s: live_samples must be 4-byte aligned", what);
        MVSN_REQUIRE(reinterpret_cast<uintptr_t>(stop->tiles_done) % 8 == 0, MVSN_EALIGN,
                     "%s: tiles_done must be 8-byte aligned", what);
    }
    MVSN_REQUIRE(N >= 0 && S > 0, MVSN_EBADSHAPE, "%s: N=%d S=%d", what, N, S);
    MVSN_REQUIRE(S <= 128, MVSN_EUNSUPPORTED, "%s: N_samples=%d > 128 is not implemented", what, S);
    MVSN_REQUIRE(scene->mlp_mode == MVSN_MLP_FP32, MVSN_EUNSUPPORTED,
                 "%s: scene->mlp_packed must be the MVSN_MLP_FP32 image (mode %d given)", what, scene->mlp_mode);
    if (N == 0) return MVSN_OK;
    RenderIO io{};
    io.pts = in.pts; io.ndc = in.ndc; io.z = in.z; io.dirs = in.dirs;
    io.rays = in.rays; io.t_steps = in.t_steps;
    if (rays) io.rg = make_ray_gen(scene, in.rp);
    io.N = N; io.S = S;
    const BwdCall call{what, g, mlp_w, grad_mlp, grad_volume_dhwc, workspace, workspace_bytes, grad_mode, det, in.jitter,
                       stop};
    return launch_render_backward(sc, io, static_cast<const float*>(scene->mlp_packed), call, (cudaStream_t)stream);
}

size_t mvsn_render_backward_workspace_bytes(int N, int S) {
    return backward_bytes(false, N, S, 0, 0, 0, MVSN_MLP_FP32, false, false);
}
int mvsn_render_backward(const mvsn_render_scene* scene, const float* const* mlp_w, const float* rays_pts,
                         const float* rays_ndc, const float* z_vals, const float* rays_dir, int N, int S,
                         const mvsn_render_grads* g, float* const* grad_mlp, float* grad_volume_dhwc, void* workspace,
                         size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_render_backward");
    return backward_entry("mvsn_render_backward", false, scene, mlp_w, {rays_pts, rays_ndc, z_vals, rays_dir}, N, S,
                          MVSN_MLP_FP32, false, nullptr, g, grad_mlp, grad_volume_dhwc, workspace, workspace_bytes, stream);
}

size_t mvsn_render_backward_tc_workspace_bytes(int N, int S) {
    return backward_bytes(false, N, S, 0, 0, 0, MVSN_MLP_TC_HALF, false, false);
}
int mvsn_render_backward_tc(const mvsn_render_scene* scene, const float* const* mlp_w, const float* rays_pts,
                            const float* rays_ndc, const float* z_vals, const float* rays_dir, int N, int S,
                            const mvsn_render_grads* g, float* const* grad_mlp, float* grad_volume_dhwc, void* workspace,
                            size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_render_backward_tc");
    return backward_entry("mvsn_render_backward_tc", false, scene, mlp_w, {rays_pts, rays_ndc, z_vals, rays_dir}, N, S,
                          MVSN_MLP_TC_HALF, false, nullptr, g, grad_mlp, grad_volume_dhwc, workspace, workspace_bytes,
                          stream);
}

size_t mvsn_render_backward_deterministic_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode) {
    return backward_bytes(false, N, S, D, Hp, Wp, grad_mode, true, false);
}
int mvsn_render_backward_deterministic(const mvsn_render_scene* scene, const float* const* mlp_w, const float* rays_pts,
                                       const float* rays_ndc, const float* z_vals, const float* rays_dir, int N, int S,
                                       int grad_mode, const mvsn_render_grads* g, float* const* grad_mlp,
                                       float* grad_volume_dhwc, void* workspace, size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_render_backward_deterministic");
    return backward_entry("mvsn_render_backward_deterministic", false, scene, mlp_w,
                          {rays_pts, rays_ndc, z_vals, rays_dir}, N, S, grad_mode, true, nullptr, g, grad_mlp,
                          grad_volume_dhwc, workspace, workspace_bytes, stream);
}

size_t mvsn_render_backward_stop_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode, int deterministic) {
    return backward_bytes(false, N, S, D, Hp, Wp, grad_mode, deterministic != 0, true);
}
int mvsn_render_backward_stop(const mvsn_render_scene* scene, const float* const* mlp_w, const float* rays_pts,
                              const float* rays_ndc, const float* z_vals, const float* rays_dir, int N, int S,
                              int grad_mode, int deterministic, float t_stop, const mvsn_render_grads* g,
                              float* const* grad_mlp, float* grad_volume_dhwc, int* live_samples,
                              unsigned long long* tiles_done, void* workspace, size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_render_backward_stop");
    const BwdStop stop{t_stop, live_samples, tiles_done};
    return backward_entry("mvsn_render_backward_stop", false, scene, mlp_w, {rays_pts, rays_ndc, z_vals, rays_dir}, N, S,
                          grad_mode, deterministic != 0, &stop, g, grad_mlp, grad_volume_dhwc, workspace,
                          workspace_bytes, stream);
}

size_t mvsn_render_backward_rays_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode, int deterministic) {
    return backward_bytes(true, N, S, D, Hp, Wp, grad_mode, deterministic != 0, false);
}
int mvsn_render_backward_rays(const mvsn_render_scene* scene, const float* const* mlp_w, const mvsn_ray_params* rp,
                              const float* rays, const float* t_steps, const float* jitter, int N, int S, int grad_mode,
                              int deterministic, const mvsn_render_grads* g, float* const* grad_mlp,
                              float* grad_volume_dhwc, void* workspace, size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_render_backward_rays");
    return backward_entry("mvsn_render_backward_rays", true, scene, mlp_w,
                          {nullptr, nullptr, nullptr, nullptr, rp, rays, t_steps, jitter}, N, S, grad_mode,
                          deterministic != 0, nullptr, g, grad_mlp, grad_volume_dhwc, workspace, workspace_bytes, stream);
}

size_t mvsn_render_backward_rays_stop_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode, int deterministic) {
    return backward_bytes(true, N, S, D, Hp, Wp, grad_mode, deterministic != 0, true);
}
int mvsn_render_backward_rays_stop(const mvsn_render_scene* scene, const float* const* mlp_w, const mvsn_ray_params* rp,
                                   const float* rays, const float* t_steps, const float* jitter, int N, int S,
                                   int grad_mode, int deterministic, float t_stop, const mvsn_render_grads* g,
                                   float* const* grad_mlp, float* grad_volume_dhwc, int* live_samples,
                                   unsigned long long* tiles_done, void* workspace, size_t workspace_bytes, void* stream) {
    MVSN_RANGE("mvsn_render_backward_rays_stop");
    const BwdStop stop{t_stop, live_samples, tiles_done};
    return backward_entry("mvsn_render_backward_rays_stop", true, scene, mlp_w,
                          {nullptr, nullptr, nullptr, nullptr, rp, rays, t_steps, jitter}, N, S, grad_mode,
                          deterministic != 0, &stop, g, grad_mlp, grad_volume_dhwc, workspace, workspace_bytes, stream);
}

int mvsn_adam_step(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                   const int* numel_host, int count, float lr, float beta1, float beta2, float eps, int step,
                   void* stream) {
    MVSN_RANGE("mvsn_adam_step");
    MVSN_REQUIRE(params && grads && exp_avg && exp_avg_sq && numel_host, MVSN_ENULL, "mvsn_adam_step: NULL argument");
    MVSN_REQUIRE(step >= 1, MVSN_EBADSHAPE, "mvsn_adam_step: step=%d (counts from 1)", step);
    return launch_adam_tensors(params, grads, exp_avg, exp_avg_sq, numel_host, count, lr, beta1, beta2, eps, step,
                               (cudaStream_t)stream);
}

int mvsn_adam_step_volume(float* param, float* grad_dhwc, float* exp_avg, float* exp_avg_sq, long long nvox,
                          int planar, float lr, float beta1, float beta2, float eps, int step, void* stream) {
    MVSN_RANGE("mvsn_adam_step_volume");
    MVSN_REQUIRE(param && grad_dhwc && exp_avg && exp_avg_sq, MVSN_ENULL, "mvsn_adam_step_volume: NULL argument");
    MVSN_REQUIRE(nvox > 0 && step >= 1, MVSN_EBADSHAPE, "mvsn_adam_step_volume: nvox=%lld step=%d", nvox, step);
    MVSN_REQUIRE(aligned16(grad_dhwc) && (planar || (aligned16(param) && aligned16(exp_avg) && aligned16(exp_avg_sq))),
                 MVSN_EALIGN, "mvsn_adam_step_volume: buffers must be 16-byte aligned");
    return launch_adam_volume(param, grad_dhwc, exp_avg, exp_avg_sq, nvox, planar, lr, beta1, beta2, eps, step,
                              (cudaStream_t)stream);
}

// ---- exportable frame buffers (CUDA IPC): the one allocation this library makes --------------------------
int mvsn_peer_buffer_create(size_t bytes, void** dev_ptr, unsigned char* handle_host) {
    MVSN_REQUIRE(dev_ptr && handle_host && bytes > 0, MVSN_ENULL, "mvsn_peer_buffer_create: bad argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == MVSN_PEER_HANDLE_BYTES, "IPC handle size");
    void* p = nullptr;
    MVSN_CUDA_CHECK(cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        set_error("cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
        return MVSN_ECUDA;
    }
    memcpy(handle_host, &h, sizeof(h));
    *dev_ptr = p;
    return MVSN_OK;
}

int mvsn_peer_buffer_open(const unsigned char* handle_host, void** peer_ptr) {
    MVSN_REQUIRE(handle_host && peer_ptr, MVSN_ENULL, "mvsn_peer_buffer_open: NULL argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle_host, sizeof(h));
    MVSN_CUDA_CHECK(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return MVSN_OK;
}

int mvsn_peer_buffer_close(void* peer_ptr) {
    if (peer_ptr) MVSN_CUDA_CHECK(cudaIpcCloseMemHandle(peer_ptr));
    return MVSN_OK;
}

int mvsn_peer_buffer_destroy(void* dev_ptr) {
    if (dev_ptr) MVSN_CUDA_CHECK(cudaFree(dev_ptr));
    return MVSN_OK;
}

}  // extern "C"
