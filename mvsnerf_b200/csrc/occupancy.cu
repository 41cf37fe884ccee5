// K-C empty-space skipping: the occupancy grid of a scene's density (mvsn_build_occupancy) and the per-group tile
// ranges the STOP render kernels take from it (mvsn_render_rays_occ).
//
// Grid: one bit per cell of the encoding volume's D x Hp x Wp node grid in NDC, bit c = (d * Hp + y) * Wp + x of word
// c / 32 (LSB first).  Cell (d, y, x), d < D - 1, y < Hp - 1, x < Wp - 1, spans nodes d..d+1, y..y+1, x..x+1; the bits
// of the last slab in each axis are 0 and never read.  A cell is occupied when alpha = 1 - exp(-sigma) > 0 at any of its
// eight corner nodes, sigma evaluated by the split-mode samples entry with the node as the sample's NDC, then dilated by
// a (2 dilate + 1)^3 box.  sigma depends on the position only (the view direction enters the colour head alone), so a
// grid serves every view of the scene.
//
// Density grid (mvsn_build_density, the importance sampler's input): sigma itself, fp32, at every node, laid out
// [D][Hp][Wp] -- the same node samples, evaluated by the fp32 forward tile (tile_fp32.cuh) that the FFMA render and the
// fine-tuning backward share, which leaves sigma = relu(alpha_linear(h)) before any exponential.
#include "tile_fp32.cuh"

namespace mvsn {

namespace occ {
constexpr int CHUNK_SAMPLES = 1 << 20;                    // nodes per samples-entry launch
constexpr int MAX_DILATE = 8;
static size_t round16(size_t b) { return (b + 15) & ~(size_t)15; }
static long long nodes(int D, int Hp, int Wp) { return (long long)D * Hp * Wp; }
static int chunk_rows(int D, int Hp, int Wp) {
    const int r = CHUNK_SAMPLES / Wp;
    return r < 1 ? 1 : r > D * Hp ? D * Hp : r;
}
}  // namespace occ

size_t occupancy_words(int D, int Hp, int Wp) { return (size_t)((occ::nodes(D, Hp, Wp) + 31) / 32); }

// workspace: alpha [nodes] fp32 | two cell byte maps [nodes] | one chunk of samples: pts [R*Wp,3], ndc [R*Wp,3],
// z [R*Wp], dirs [R,3]
size_t occupancy_workspace_bytes(int D, int Hp, int Wp) {
    if (D < 2 || Hp < 2 || Wp < 2) return 0;
    const size_t n = (size_t)occ::nodes(D, Hp, Wp), cs = (size_t)occ::chunk_rows(D, Hp, Wp) * Wp;
    return occ::round16(n * 4) + 2 * occ::round16(n) + 2 * occ::round16(cs * 12) + occ::round16(cs * 4) +
           occ::round16((size_t)occ::chunk_rows(D, Hp, Wp) * 12);
}

// The samples of rows [row0, row0 + rows) of the node grid (row = d * Hp + y, sample = x): ndc = the node (x / (Wp - 1),
// y / (Hp - 1), d / (D - 1)), the world point ndc_of_point inverts to (pad, lindisp, the reference camera), z = 0 and a
// unit direction (neither enters sigma).  (K R)^-1 and K t are formed once per block in double.
__global__ void occ_nodes_kernel(const SceneDev sc, const RayGenDev rg, int row0, int rows, float* __restrict__ pts,
                                 float* __restrict__ ndc, float* __restrict__ z, float* __restrict__ dirs) {
    __shared__ double minv[9], kt[3];
    if (threadIdx.x == 0) {
        double R[9], K[9], t[3], M[9];
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) { R[3 * i + j] = sc.w2cs[4 * i + j]; K[3 * i + j] = sc.intrinsics[3 * i + j]; }
            t[i] = sc.w2cs[4 * i + 3];
        }
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) M[3 * i + j] = K[3 * i] * R[j] + K[3 * i + 1] * R[3 + j] + K[3 * i + 2] * R[6 + j];
        for (int i = 0; i < 3; ++i) kt[i] = K[3 * i] * t[0] + K[3 * i + 1] * t[1] + K[3 * i + 2] * t[2];
        const double det = M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) +
                           M[2] * (M[3] * M[7] - M[4] * M[6]);
        const double id = 1.0 / det;
        minv[0] = (M[4] * M[8] - M[5] * M[7]) * id; minv[1] = (M[2] * M[7] - M[1] * M[8]) * id;
        minv[2] = (M[1] * M[5] - M[2] * M[4]) * id; minv[3] = (M[5] * M[6] - M[3] * M[8]) * id;
        minv[4] = (M[0] * M[8] - M[2] * M[6]) * id; minv[5] = (M[2] * M[3] - M[0] * M[5]) * id;
        minv[6] = (M[3] * M[7] - M[4] * M[6]) * id; minv[7] = (M[1] * M[6] - M[0] * M[7]) * id;
        minv[8] = (M[0] * M[4] - M[1] * M[3]) * id;
    }
    __syncthreads();
    const int Wp = sc.Wp, Hp = sc.Hp;
    const long long n = (long long)rows * Wp;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int r = row0 + (int)(i / Wp), x = (int)(i % Wp), d = r / Hp, y = r % Hp;
        const float nx = __fdiv_rn((float)x, (float)(Wp - 1)), ny = __fdiv_rn((float)y, (float)(Hp - 1)),
                    nz = __fdiv_rn((float)d, (float)(sc.D - 1));
        double u = nx, v = ny;
        if (rg.pad > 0.f) {                                   // utils.py:140-143 undone
            const double dw = (double)rg.wf + 2.0 * rg.pad, dh = (double)rg.hf + 2.0 * rg.pad;
            u = (u * dw - rg.pad) / rg.wf;
            v = (v * dh - rg.pad) / rg.hf;
        }
        const double zc = rg.lindisp ? 1.0 / ((double)rg.inv_near + (double)nz * rg.inv_far_minus_inv_near)
                                     : (double)rg.near + (double)nz * rg.far_minus_near;
        const double q[3] = {u * (sc.W - 1) * zc - kt[0], v * (sc.H - 1) * zc - kt[1], zc - kt[2]};
        for (int j = 0; j < 3; ++j) {
            pts[3 * i + j] = (float)(minv[3 * j] * q[0] + minv[3 * j + 1] * q[1] + minv[3 * j + 2] * q[2]);
        }
        ndc[3 * i] = nx; ndc[3 * i + 1] = ny; ndc[3 * i + 2] = nz;
        z[i] = 0.f;
        if (x == 0) { dirs[3 * (i / Wp)] = 0.f; dirs[3 * (i / Wp) + 1] = 0.f; dirs[3 * (i / Wp) + 2] = 1.f; }
    }
}

// cell (d, y, x) of the first three axes' first n - 1 nodes: 1 when alpha > 0 at any of its eight corner nodes
__global__ void occ_cells_kernel(const float* __restrict__ alpha, int D, int Hp, int Wp, uint8_t* __restrict__ cells) {
    const long long n = (long long)D * Hp * Wp;
    for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < n; c += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(c % Wp), y = (int)((c / Wp) % Hp), d = (int)(c / ((long long)Wp * Hp));
        bool o = false;
        if (d < D - 1 && y < Hp - 1 && x < Wp - 1) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const long long node = c + ((k >> 2) ? (long long)Hp * Wp : 0) + (((k >> 1) & 1) ? Wp : 0) + (k & 1);
                o |= __ldg(alpha + node) > 0.f;
            }
        }
        cells[c] = o;
    }
}

// one axis of the box dilation: out[c] = any in[c + k * stride], |k| <= r, over the axis' valid cells [0, len - 2]
__global__ void occ_dilate_kernel(const uint8_t* __restrict__ in, int D, int Hp, int Wp, int axis, int r,
                                  uint8_t* __restrict__ out) {
    const long long n = (long long)D * Hp * Wp;
    const long long stride = axis == 0 ? 1 : axis == 1 ? Wp : (long long)Wp * Hp;
    const int len = axis == 0 ? Wp : axis == 1 ? Hp : D;
    for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < n; c += (long long)gridDim.x * blockDim.x) {
        const int p = (int)((c / stride) % len);
        bool o = false;
        if (p < len - 1) {
            const int lo = p - r < 0 ? 0 : p - r, hi = p + r > len - 2 ? len - 2 : p + r;
            for (int q = lo; q <= hi && !o; ++q) o = in[c + (q - p) * stride] != 0;
        }
        out[c] = o;
    }
}

// byte map -> bits (32 consecutive cells per word, one warp per word)
__global__ void occ_pack_kernel(const uint8_t* __restrict__ cells, long long n, uint32_t* __restrict__ bits) {
    const long long total = (n + 31) / 32 * 32;
    for (long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
        const uint32_t w = __ballot_sync(0xffffffffu, c < n && cells[c] != 0);
        if ((threadIdx.x & 31) == 0) bits[c >> 5] = w;
    }
}

static int grid_of(long long n) { return cdiv(n, 256) < 8192 ? cdiv(n, 256) : 8192; }

int build_occupancy(const SceneDev& sc, const RayGenDev& rg, const void* wimg_split, bool half_vol, int dilate,
                    uint32_t* bits, void* workspace, cudaStream_t stream) {
    const int D = sc.D, Hp = sc.Hp, Wp = sc.Wp;
    const long long n = occ::nodes(D, Hp, Wp);
    const int R = occ::chunk_rows(D, Hp, Wp);
    const size_t cs = (size_t)R * Wp;
    uint8_t* p = static_cast<uint8_t*>(workspace);
    float* alpha = reinterpret_cast<float*>(p);                 p += occ::round16(n * 4);
    uint8_t* cell_a = p;                                        p += occ::round16(n);
    uint8_t* cell_b = p;                                        p += occ::round16(n);
    float* pts = reinterpret_cast<float*>(p);                   p += occ::round16(cs * 12);
    float* ndc = reinterpret_cast<float*>(p);                   p += occ::round16(cs * 12);
    float* z = reinterpret_cast<float*>(p);                     p += occ::round16(cs * 4);
    float* dirs = reinterpret_cast<float*>(p);
    for (int row0 = 0; row0 < D * Hp; row0 += R) {
        const int rows = D * Hp - row0 < R ? D * Hp - row0 : R;
        occ_nodes_kernel<<<grid_of((long long)rows * Wp), 256, 0, stream>>>(sc, rg, row0, rows, pts, ndc, z, dirs);
        MVSN_CUDA_CHECK(cudaGetLastError());
        RenderIO io{};                                          // the samples entry: one "ray" per node row
        io.pts = pts; io.ndc = ndc; io.z = z; io.dirs = dirs;
        io.N = rows; io.S = Wp;
        io.alpha = alpha + (size_t)row0 * Wp;
        const int rc = launch_render_wg(sc, io, false, true, wimg_split, stream, nullptr, nullptr, half_vol);
        if (rc) return rc;
    }
    occ_cells_kernel<<<grid_of(n), 256, 0, stream>>>(alpha, D, Hp, Wp, cell_a);
    MVSN_CUDA_CHECK(cudaGetLastError());
    uint8_t* cur = cell_a;
    if (dilate > 0) {
        uint8_t* other = cell_b;
        for (int axis = 0; axis < 3; ++axis) {
            occ_dilate_kernel<<<grid_of(n), 256, 0, stream>>>(cur, D, Hp, Wp, axis, dilate, other);
            MVSN_CUDA_CHECK(cudaGetLastError());
            uint8_t* t = cur; cur = other; other = t;
        }
    }
    occ_pack_kernel<<<grid_of(n), 256, 0, stream>>>(cur, n, bits);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

// ------------------------------------------------------------------------------------------------
// density grid
// ------------------------------------------------------------------------------------------------
// sigma of the io.N x io.S node samples occ_nodes_kernel wrote (sample i = ray i / S, step i % S): 128 consecutive
// samples per tile, tiles strided over the CTAs.  VT = __half: sc.vol is the fp16 image (sample_volume<__half>), so the
// grid equals the one of the volume vol.half().float() bit for bit.
template <typename VT>
__global__ void __launch_bounds__(256, 1) density_tile_kernel(const SceneDev sc, const RenderIO io,
                                                               const float* __restrict__ wts, float* __restrict__ sigma) {
    extern __shared__ __align__(16) float smem[];
    const TileSmem sm(smem);
    const int tid = threadIdx.x;
    __shared__ Cams cams;
    load_cams(sc, &cams, tid);
    __syncthreads();
    const long long n = (long long)io.N * io.S, ntiles = (n + TILE_M - 1) / TILE_M;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const long long i = t * TILE_M + tid;
        const bool valid = tid < TILE_M && i < n;
        if (tid < TILE_M)
            tile_front_end<false, NoRecord, VT>(sc, cams, io, sm, tid, valid ? (int)(i / io.S) : 0,
                                                valid ? (int)(i % io.S) : 0, valid, NoRecord{});
        __syncthreads();
        tile_mlp(sm, wts, tid, NoRecord{});
        if (valid) sigma[i] = sm.sig[tid];                     // written by this thread inside tile_mlp
        __syncthreads();
    }
}

// workspace: one chunk of node samples, laid out as build_occupancy's
size_t density_workspace_bytes(int D, int Hp, int Wp) {
    if (D < 2 || Hp < 2 || Wp < 2) return 0;
    const size_t cs = (size_t)occ::chunk_rows(D, Hp, Wp) * Wp;
    return 2 * occ::round16(cs * 12) + occ::round16(cs * 4) + occ::round16((size_t)occ::chunk_rows(D, Hp, Wp) * 12);
}

int build_density(const SceneDev& sc, const RayGenDev& rg, const float* wts_fp32, bool half_vol, float* sigma,
                  void* workspace, cudaStream_t stream) {
    constexpr int SMEM = TILE_SMEM_FLOATS * sizeof(float);
    static bool attr_set[64] = {false};                   // once per device, not per launch
    int dev = 0;
    MVSN_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !attr_set[dev]) {
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(density_tile_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        MVSN_CUDA_CHECK(cudaFuncSetAttribute(density_tile_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        if (dev < 64) attr_set[dev] = true;
    }
    const int D = sc.D, Hp = sc.Hp, Wp = sc.Wp;
    const int R = occ::chunk_rows(D, Hp, Wp);
    const size_t cs = (size_t)R * Wp;
    uint8_t* p = static_cast<uint8_t*>(workspace);
    float* pts = reinterpret_cast<float*>(p);                   p += occ::round16(cs * 12);
    float* ndc = reinterpret_cast<float*>(p);                   p += occ::round16(cs * 12);
    float* z = reinterpret_cast<float*>(p);                     p += occ::round16(cs * 4);
    float* dirs = reinterpret_cast<float*>(p);
    for (int row0 = 0; row0 < D * Hp; row0 += R) {
        const int rows = D * Hp - row0 < R ? D * Hp - row0 : R;
        occ_nodes_kernel<<<grid_of((long long)rows * Wp), 256, 0, stream>>>(sc, rg, row0, rows, pts, ndc, z, dirs);
        MVSN_CUDA_CHECK(cudaGetLastError());
        RenderIO io{};
        io.pts = pts; io.ndc = ndc; io.z = z; io.dirs = dirs;
        io.N = rows; io.S = Wp;
        const long long tiles = ((long long)rows * Wp + TILE_M - 1) / TILE_M;
        const int grid = tiles < sm_count() ? (int)tiles : sm_count();
        float* out = sigma + (size_t)row0 * Wp;
        if (half_vol) density_tile_kernel<__half><<<grid, 256, SMEM, stream>>>(sc, io, wts_fp32, out);
        else          density_tile_kernel<float><<<grid, 256, SMEM, stream>>>(sc, io, wts_fp32, out);
        MVSN_CUDA_CHECK(cudaGetLastError());
    }
    return MVSN_OK;
}

// ------------------------------------------------------------------------------------------------
// per-group tile ranges of a ray launch
// ------------------------------------------------------------------------------------------------
// whether sample (ray, s) lies in an occupied cell; outside [0,1]^3 (or NaN) counts as occupied.  PRECISE: the NDC of
// the render kernel's front end in that mode (sample_point<true, PRECISE>), so the samples are the ones it computes.
template <bool PRECISE>
__device__ __forceinline__ bool sample_occupied(const SceneDev& sc, const Cams& cams, const RenderIO& io,
                                                const uint32_t* __restrict__ bits, int ray, int s) {
    float px, py, pz, dx, dy, dz, nx, ny, nz, z;
    sample_point<true, PRECISE>(sc, cams, io, ray, s, (size_t)ray * io.S + s, px, py, pz, dx, dy, dz, nx, ny, nz, z);
    if (!(nx >= 0.f && nx <= 1.f && ny >= 0.f && ny <= 1.f && nz >= 0.f && nz <= 1.f)) return true;
    const Trilinear t = trilinear_corners(sc, nx, ny, nz);
    const int x = min(t.x0, sc.Wp - 2), y = min(t.y0, sc.Hp - 2), d = min(t.z0, sc.D - 2);
    const long long c = ((long long)d * sc.Hp + y) * sc.Wp + x;
    return (__ldg(bits + (c >> 5)) >> (c & 31)) & 1u;
}

// One thread per ray (a warp holds 32 / RT whole groups): the first and the last sample in an occupied cell, as tiles
// (tile = s / SP), reduced over the group's RT lanes -> ranges[g] = (k_first, k_last); (NT, -1) when no sample of the
// group is occupied, and the group's pixels are stored here as the full render stores them when every alpha is 0.
template <bool PRECISE>
__global__ void __launch_bounds__(256) occ_ranges_kernel(const SceneDev sc, const RenderIO io,
                                                         const uint32_t* __restrict__ bits, int2* __restrict__ ranges) {
    __shared__ Cams cams;
    load_cams(sc, &cams, threadIdx.x);
    __syncthreads();
    const int RT = io.rays_per_tile, SP = 64 / RT, S = io.S, N = io.N;
    const int NT = (S + SP - 1) / SP, G = (N + RT - 1) / RT;
    const int ray = blockIdx.x * blockDim.x + threadIdx.x;
    int first = S, last = -1;
    if (ray < N) {
        for (int s = 0; s < S; ++s)
            if (sample_occupied<PRECISE>(sc, cams, io, bits, ray, s)) { first = s; break; }
        for (int s = S - 1; s >= first; --s)
            if (sample_occupied<PRECISE>(sc, cams, io, bits, ray, s)) { last = s; break; }
    }
    int kf = first < S ? first / SP : NT, kl = last >= 0 ? last / SP : -1;
    for (int o = 1; o < RT; o <<= 1) {
        kf = min(kf, __shfl_xor_sync(0xffffffffu, kf, o));
        kl = max(kl, __shfl_xor_sync(0xffffffffu, kl, o));
    }
    const int grp = ray / RT;
    if ((ray & (RT - 1)) == 0 && grp < G) {
        ranges[grp] = make_int2(kf, kl);
        if (kl < 0) {                                           // c0..c4 = 0: rgb 0 (white_bkgd: 0 + (1 - 0)), depth 0
            const float bg = sc.white_bkgd ? 1.f : 0.f;
            for (int r = grp * RT; r < grp * RT + RT && r < N; ++r) store_pixel(io, r, bg, bg, bg, 0.f);
        }
    }
}

size_t occupancy_ranges_bytes(int N) { return occ::round16((size_t)((N + 3) / 4) * sizeof(int2)); }

int launch_occupancy_ranges(const SceneDev& sc, const RenderIO& io, bool precise, const uint32_t* bits, int2* ranges,
                            cudaStream_t stream) {
    const int grid = cdiv(io.N, 256);
    if (precise) occ_ranges_kernel<true><<<grid, 256, 0, stream>>>(sc, io, bits, ranges);
    else         occ_ranges_kernel<false><<<grid, 256, 0, stream>>>(sc, io, bits, ranges);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

}  // namespace mvsn
