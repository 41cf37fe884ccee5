// K-C, tensor-core modes (MVSN_MLP_TC_HALF / TC_PAIR: fp16 operands; MVSN_MLP_TC_SPLIT: 2-term fp16 split,
// fp32-grade): the fused per-ray render kernel with the per-sample MLP on Hopper warpgroup MMAs (wgmma,
// fp32 accumulators in registers).
//
// One persistent CTA per SM.  fp16-operand modes, warp-specialised (NWG + 2 roles):
//   warpgroups 0..NWG-1  consumers, one 64-sample tile each: the eight GEMM phases of the MLP, their epilogues
//                        and the alpha compositing.  The accumulator fragment of a layer, after bias, modulation
//                        and ReLU, is converted in registers into the A operand of the next layer (the wgmma
//                        accumulator and register-A layouts coincide), so hidden activations never touch
//                        shared memory.
//   warpgroup NWG        producer: the per-sample front end (ray march, NDC, trilinear + colour gather,
//                        positional encoding) of the consumers' upcoming tiles, two threads per sample row,
//                        into a ring of operand-tile slots (PE | MISC, two slots per consumer, full / empty
//                        mbarriers).  The MMA warpgroups never wait on gathers, and the front end of one tile
//                        overlaps the GEMMs and epilogues of the others.
//   last warp            weight loader: one thread streams the weight image, one K-block of one layer at a
//                        time, L2 -> a shared-memory ring with 1-D bulk async copies (mbarrier complete_tx);
//                        every consumer consumes the same chunk sequence.  fp16 without STOP: half of the image
//                        (RES_MASK) is copied once and stays resident; only the other chunks are streamed.
// Split mode (hi | lo operands, twice the operand bytes) does not fit the slot ring in shared memory, so there
// every warpgroup runs its own front end before its GEMMs (NWG + 1 roles, no producer).
// feature_linear has no non-linearity before views_linears[0] (models.py:213-218): the two are folded at pack
// time (fp64) into one GEMM from h, with alpha_linear as one extra output row.  Biases are added in fp32 in the
// epilogues.  Split mode: every operand is x = hi + lo (fp16), three MMAs per K-step (hi*lo + lo*hi + hi*hi),
// with exact power-of-two scales, undone in the epilogues:
//   front-end operands (encoding, features, view direction)  none: |x| < 65504
//   weights                                                   2^ew for the whole image: x256, lowered when the largest
//                                                             |w| reaches 128 so that it packs below 2^15
//   hidden activations                                        2^e per sample row, chosen by the epilogue that makes the
//                                                             row: its maximum lands in [2^14, 2^15), whatever the range
// The four threads of a quad hold a whole accumulator row, so the row maximum costs two shuffles, and the same thread
// holds that row in the next GEMM's accumulator.  Where one GEMM reads front-end columns and register columns (layer 5,
// folded head), the fp32 accumulator rows are rescaled exactly between the two groups of K-blocks.
//
// Replaces renderer.rendering (renderer.py:138-165) and callees; see include/mvsnerf_b200.h.
#include "render_frontend.cuh"
#include "hopper.cuh"

namespace mvsn {

using namespace hop;

namespace wg {
constexpr int NWG = 2;                                     // MMA warpgroups (tiles in flight) per CTA
// Three schedules:
//   fp16 without STOP (rmod): the modulation lives in the consumers' registers.  NWG consumers + the producer
//        warpgroup + a loader warpgroup (its first warp loads, the other three leave at once); setmaxnreg moves the
//        producer's and the loader's registers to the consumers.
//   fp16 with STOP: the modulation in shared memory; NWG consumers + the producer + the loader warp, 128 registers
//        each.  ptxas does not allocate the STOP consumers beyond the launch budget after a setmaxnreg.inc (they
//        spill), so they keep the layout without register modulation.
//   split: NWG warpgroups + the loader warp.
__host__ __device__ constexpr int threads(bool split, bool rmod) {
    return split ? NWG * 128 + 32 : rmod ? (NWG + 2) * 128 : (NWG + 1) * 128 + 32;
}
__host__ __device__ constexpr int loader_warp(bool split) { return split ? NWG * 4 : (NWG + 1) * 4; }
// rmod: registers per thread of each role (launched at 65536 / 512 = 128 each).  The consumers hold acc (64) + the
// next layer's A operand (32) + the modulation (64); the sum over the four warpgroups must fit the 64 K register file.
constexpr int REGS_CONSUMER = 192, REGS_PRODUCER = 104, REGS_LOADER = 24;
static_assert((NWG * REGS_CONSUMER + REGS_PRODUCER + REGS_LOADER) * 128 <= 65536, "register file");
constexpr int ROWS = 64;                                   // samples per tile
constexpr int NCHUNK = 17;
// B-operand rows of each chunk (one 64-wide K-block of one layer, consumption order):
//  0 pts_bias | 1 layer 0 | 2-9 layers 1-4 (two K-blocks each) | 10 layer 5, encoding part | 11-12 layer 5, h part
//  13-14 folded head from h (64 views rows + alpha) | 15 folded head, view-direction part | 16 rgb
__host__ __device__ constexpr int chunk_rows(int c) { return c >= 13 && c <= 15 ? 72 : c == 16 ? 8 : 128; }
constexpr int HALF_STRIDE = 16384;                         // bytes of one fp16 image of a chunk (hi; lo follows in split mode)
__host__ __device__ constexpr int chunk_stride(bool split) { return split ? 2 * HALF_STRIDE : HALF_STRIDE; }
// fp32 bias tail after the chunks; split mode also keeps there the largest |weight| (fp32 bits) and 2^-ew
constexpr int BIAS_MOD = 0, BIAS_TRUNK = 128, BIAS_HEAD = 896, BIAS_RGB = 968, BIAS_WINV = 1016, BIAS_WMAX = 1017,
              BIAS_FLOATS = 1024;
__host__ __device__ constexpr int tail_offset(bool split) { return NCHUNK * chunk_stride(split); }
__host__ __device__ constexpr int image_bytes(bool split) { return tail_offset(split) + BIAS_FLOATS * 4; }
// rmod: the chunks that stay resident in shared memory for the whole kernel (copied once per CTA): the modulation,
// layer 0, the folded head, rgb and three trunk chunks spread between the streamed ones.  The other eight chunks
// (128 KB per pass instead of 236) are streamed through the ring.
constexpr uint32_t RES_MASK = 0x3u | (1u << 4) | (1u << 7) | (1u << 10) | 0x1E000u;
__host__ __device__ constexpr bool resident(int c) { return (RES_MASK >> c) & 1u; }
static_assert((RES_MASK >> 13) == 0xFu, "the folded head and rgb are resident");
__host__ __device__ constexpr uint32_t popc32(uint32_t x) {
    x = x - ((x >> 1) & 0x55555555u);
    x = (x & 0x33333333u) + ((x >> 2) & 0x33333333u);
    return (((x + (x >> 4)) & 0x0F0F0F0Fu) * 0x01010101u) >> 24;
}
// byte offset of resident chunk c in the resident region: the resident chunks in order, the 128-row ones (16 KB) before
// the head's 72-row ones (9 KB) -- multiples of the 1024 that SW128 tiles need
__host__ __device__ constexpr uint32_t res_offset(int c) {
    return 16384u * popc32(RES_MASK & ((1u << (c < 13 ? c : 13)) - 1u)) + 9216u * (c > 13 ? c - 13 : 0);
}
constexpr int NSTREAM = NCHUNK - (int)popc32(RES_MASK), RES_BYTES = (int)res_offset(NCHUNK - 1) + 1024;
// shared memory
//   split:       per warpgroup [PE (hi | lo) | MISC (hi | lo) | modulation fp32 | exchange], the ring (2 stages), the biases
//   fp16 rmod:   SLOTS operand-tile slots [PE | MISC], per consumer an exchange, the ring (2 stages), the resident
//                chunks, the biases = 64 + 2 x 1 + 32 + 108 + 4 KB (+ 1 KB alignment) = 211 KB
//   fp16 STOP:   SLOTS operand-tile slots, per consumer [modulation fp32 | exchange], the ring (4 stages), the biases
//                = 64 + 2 x 33 + 64 + 4 KB (+ 1 KB alignment) = 199 KB
__host__ __device__ constexpr int tile_bytes(bool split) { return split ? 16384 : 8192; }
__host__ __device__ constexpr int off_misc(bool split) { return tile_bytes(split); }
constexpr int MOD_BYTES = ROWS * 128 * 4, XCH_BYTES = 1024;
constexpr int SLOTS = 2 * NWG;                             // fp16: operand-tile slots, two per consumer
constexpr int SLOT_BYTES = 2 * 8192;
__host__ __device__ constexpr int off_mod(bool split) { return 2 * tile_bytes(split); }   // split: inside a warpgroup's region
__host__ __device__ constexpr int wg_bytes(bool split) { return off_mod(split) + MOD_BYTES + XCH_BYTES; }
// [modulation |] exchange of warpgroup w (rmod: the exchange alone)
__host__ __device__ constexpr int off_state(bool split, bool rmod, int w) {
    return split ? w * wg_bytes(true) + off_mod(true) : SLOTS * SLOT_BYTES + w * ((rmod ? 0 : MOD_BYTES) + XCH_BYTES);
}
__host__ __device__ constexpr int nstage(bool split, bool rmod) { return split ? 2 : rmod ? 2 : 4; }
// entries of the static ring barrier arrays: split keeps the four and fp16 the eight of their earlier layouts, so the
// split and STOP kernels (static shared memory offsets included) stay as they were
__host__ __device__ constexpr int ring_bars(bool split) { return split ? 4 : 8; }
static_assert(nstage(true, false) <= ring_bars(true) && nstage(false, false) <= ring_bars(false) &&
              nstage(false, true) <= ring_bars(false), "ring barriers");
// rmod: a consumer takes the streamed stages of a whole layer before its first wgmma (trunk layers 1-5: chunks 2-3,
// 4-5, 6-7, 8-9, 10-12), so the ring must hold them
static_assert(popc32(~RES_MASK & 0xCu) <= nstage(false, true) && popc32(~RES_MASK & 0x30u) <= nstage(false, true) &&
              popc32(~RES_MASK & 0xC0u) <= nstage(false, true) && popc32(~RES_MASK & 0x300u) <= nstage(false, true) &&
              popc32(~RES_MASK & 0x1C00u) <= nstage(false, true), "ring depth");
__host__ __device__ constexpr int off_ring(bool split, bool rmod) {
    return split ? NWG * wg_bytes(true) : off_state(false, rmod, NWG);
}
__host__ __device__ constexpr int off_res() { return off_ring(false, true) + nstage(false, true) * HALF_STRIDE; }   // rmod
__host__ __device__ constexpr int off_bias(bool split, bool rmod) {
    return off_ring(split, rmod) + nstage(split, rmod) * chunk_stride(split) + (rmod ? RES_BYTES : 0);
}
__host__ __device__ constexpr int smem_bytes(bool split, bool rmod) { return off_bias(split, rmod) + BIAS_FLOATS * 4 + 1024; }
static_assert(smem_bytes(true, false) <= 227 * 1024, "shared memory budget");
static_assert(wg_bytes(true) % 1024 == 0 && SLOT_BYTES % 1024 == 0 && off_ring(false, true) % 1024 == 0 &&
              off_ring(false, false) % 1024 == 0 && off_res() % 1024 == 0, "SW128 tiles need 1024-byte alignment");
// early ray termination (STOP launches only, never rmod): the pass protocol's state after the biases
constexpr int STOP_BYTES = 128;
__host__ __device__ constexpr int off_stop(bool split) { return off_bias(split, false) + BIAS_FLOATS * 4; }
static_assert(smem_bytes(false, false) + STOP_BYTES <= 227 * 1024 && smem_bytes(true, false) + STOP_BYTES <= 227 * 1024,
              "shared memory budget");
}  // namespace wg

template <bool SPLIT>
struct WgShared {
    uint64_t full[wg::ring_bars(SPLIT)];                   // weight ring
    uint64_t empty[wg::ring_bars(SPLIT)];
    uint64_t slot_full[wg::SLOTS];                         // fp16: operand-tile slots
    uint64_t slot_empty[wg::SLOTS];
    Cams cams;
};
// rmod: one more barrier, for the one-shot copy of the resident chunks (appended, so the other kernels' layout stays)
struct WgSharedRes : WgShared<false> {
    uint64_t resident;
};
static_assert(wg::smem_bytes(false, true) + sizeof(WgSharedRes) <= 227 * 1024, "shared memory budget");

// STOP: every consumer publishes, at the start of pass p, what it computes in pass p + 2 (its plan); dec[(p + 2) & 3]
// completes when all consumers have (the plans of passes 0 and 1 are set up before the roles split).  The loader, the
// producer and idle consumers read the plans of a pass only after that barrier.  Four slots: a slot is rewritten two
// passes after the pass it plans, when every reader of it is provably done (see DESIGN §4 K-C).
constexpr int STOP_SLOTS = 4;
struct WgStop {
    uint64_t dec[STOP_SLOTS];
    int2 plan[STOP_SLOTS][wg::NWG];                        // (group, tile) of consumer w in pass p (slot p & 3); group -1: idle
    int next;                                              // next index into the CTA's group list
};
static_assert(sizeof(WgStop) <= wg::STOP_BYTES, "stop state");
__device__ __forceinline__ WgStop* stop_state(uint8_t* smem, bool split) { return reinterpret_cast<WgStop*>(smem + wg::off_stop(split)); }
// index j of the CTA's group list -> group: the groups the static decomposition gives this CTA, in order
__device__ __forceinline__ int stop_group(int j) {
    return ((j / wg::NWG) * (int)gridDim.x + (int)blockIdx.x) * wg::NWG + j % wg::NWG;
}
// wait for the plans of pass p >= 2 (published at the start of pass p - 2: completion (p - 2) / 4 of dec[p & 3])
__device__ __forceinline__ void stop_wait(WgStop* ss, int pass) {
    if (pass >= 2) mbar_wait(&ss->dec[pass & (STOP_SLOTS - 1)], ((pass - 2) >> 2) & 1);
}
__device__ __forceinline__ int2 stop_plan(const WgStop* ss, int pass, int w) { return ss->plan[pass & (STOP_SLOTS - 1)][w]; }
__device__ __forceinline__ bool stop_busy(const WgStop* ss, int pass, int w) { return stop_plan(ss, pass, w).x >= 0; }
__device__ __forceinline__ const int2* range_table(const int2* ranges) { return ranges; }
// the tiles [first, last] of group g that hold an occupied sample (empty-space skipping: the range table the pre-pass
// wrote; last < first: none); [0, NT - 1] without a table
__device__ __forceinline__ int2 stop_range(const int2* ranges, int g, int NT) {
    return ranges ? __ldg(ranges + g) : make_int2(0, NT - 1);
}
// the first plan (group, first tile) of the next group of the CTA's list with a non-empty range; (-1, 0) when none is
// left.  next_index() hands out the list's indices (stop_group is increasing in them).
template <typename NextIndex>
__device__ __forceinline__ int2 stop_take(const int2* ranges, NextIndex next_index, int G, int NT) {
#pragma unroll 1
    while (true) {
        const int g = stop_group(next_index());
        if (g >= G) return make_int2(-1, 0);
        const int2 r = stop_range(ranges, g, NT);
        if (r.y >= r.x) return make_int2(g, r.x);
    }
}

__device__ __forceinline__ uint32_t pack_h2_rn(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// two fp32 -> packed fp16x2 (low half = first argument), saturating: an overflow never becomes inf (inf x 0 = NaN)
__device__ __forceinline__ uint32_t cvt_h2_sat(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;\n" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
// x = hi + lo, both fp16 (x already carries the operand scale)
__device__ __forceinline__ void split_h2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
// split mode: 2^(14 - floor(log2 m)) for a row maximum m >= 0 (clamped to [2^-113, 2^54]; a zero row takes any scale)
__device__ __forceinline__ float row_scale(float m) {
    const int eb = min(max((__float_as_int(m) >> 23) & 0xff, 87), 254);
    return __int_as_float((268 - eb) << 23);
}
__device__ __forceinline__ float inv_pow2(float s) { return __int_as_float((254 << 23) - __float_as_int(s)); }
// split mode: hidden activations v (>= 0, accumulator layout: v[i] is row row_a if (i & 2) == 0, else row_b) ->
// hi / lo A registers of the next GEMM, each row scaled by sa / sb so that its maximum lies in [2^14, 2^15)
template <int NV>
__device__ __forceinline__ void split_rows(const float* v, uint32_t* ah, uint32_t* al, float& sa, float& sb) {
    float pa[4] = {0.f, 0.f, 0.f, 0.f}, pb[4] = {0.f, 0.f, 0.f, 0.f};   // four short chains per row, not one long one
#pragma unroll
    for (int j = 0; j < NV / 4; ++j) {
        pa[j & 3] = fmaxf(pa[j & 3], fmaxf(v[4 * j], v[4 * j + 1]));
        pb[j & 3] = fmaxf(pb[j & 3], fmaxf(v[4 * j + 2], v[4 * j + 3]));
    }
    float ma = fmaxf(fmaxf(pa[0], pa[1]), fmaxf(pa[2], pa[3])), mb = fmaxf(fmaxf(pb[0], pb[1]), fmaxf(pb[2], pb[3]));
    ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 1)); ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, 2));
    mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 1)); mb = fmaxf(mb, __shfl_xor_sync(0xffffffffu, mb, 2));
    sa = row_scale(ma); sb = row_scale(mb);
#pragma unroll
    for (int i = 0; i < NV; i += 2) {
        const float s = (i & 2) ? sb : sa;
        split_h2(v[i] * s, v[i + 1] * s, ah[i >> 1], al[i >> 1]);
    }
}
// split mode: the weight scale 2^ew from the largest |weight| (fp32 bits): 256 unless that would put it above 2^15
__host__ __device__ inline float weight_scale(uint32_t wmax_bits) {
    int eb = (int)(wmax_bits >> 23) & 0xff;
    eb = eb < 1 ? 1 : eb > 254 ? 254 : eb;
    const int e = 141 - eb < 8 ? 141 - eb : 8;               // 14 - floor(log2 |w|max), at most 8
    union { uint32_t u; float f; } r;
    r.u = (uint32_t)(e + 127) << 23;
    return r.f;
}

// eight consecutive operand columns (16-byte chunk c) of `row` into a SW128 tile; split: lo image 8 KB after hi
template <bool SPLIT>
__device__ __forceinline__ void store8(uint8_t* tile, int row, int c, const float* v) {
    const uint32_t off = sw128_offset(row, c * 8);
    if (SPLIT) {
        uint32_t h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) split_h2(v[2 * j], v[2 * j + 1], h[j], l[j]);
        *reinterpret_cast<uint4*>(tile + off) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(tile + 8192 + off) = make_uint4(l[0], l[1], l[2], l[3]);
    } else {
        *reinterpret_cast<uint4*>(tile + off) = make_uint4(pack_h2_rn(v[0], v[1]), pack_h2_rn(v[2], v[3]),
                                                           pack_h2_rn(v[4], v[5]), pack_h2_rn(v[6], v[7]));
    }
}

// K-steps [ks0, ks0 + nks) of one chunk with A from a shared-memory tile (split: lo 8 KB after hi; B lo 16 KB after hi)
template <int N, bool SPLIT>
__device__ __forceinline__ void gemm_ss(float (&d)[N / 2], uint32_t a, uint32_t b, int ks0, int nks, bool first) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        if (ks >= nks) break;
        const uint32_t ao = a + (ks0 + ks) * 32, bo = b + (ks0 + ks) * 32;
        const int acc = (first && ks == 0) ? 0 : 1;
        if (SPLIT) {
            Wgmma<N>::ss(d, desc_sw128(ao), desc_sw128(bo + wg::HALF_STRIDE), acc);
            Wgmma<N>::ss(d, desc_sw128(ao + 8192), desc_sw128(bo), 1);
            Wgmma<N>::ss(d, desc_sw128(ao), desc_sw128(bo), 1);
        } else {
            Wgmma<N>::ss(d, desc_sw128(ao), desc_sw128(bo), acc);
        }
    }
}
// the four K-steps of K-block `kb` with A from registers (16 registers per K-block)
template <int N, bool SPLIT>
__device__ __forceinline__ void gemm_rs(float (&d)[N / 2], const uint32_t* ah, const uint32_t* al, uint32_t b, int kb, bool first) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        const uint32_t bo = b + ks * 32;
        const int acc = (first && ks == 0) ? 0 : 1;
        const uint32_t* h = ah + (kb * 4 + ks) * 4;
        if (SPLIT) {
            const uint32_t* l = al + (kb * 4 + ks) * 4;
            Wgmma<N>::rs(d, h, desc_sw128(bo + wg::HALF_STRIDE), acc);
            Wgmma<N>::rs(d, l, desc_sw128(bo), 1);
            Wgmma<N>::rs(d, h, desc_sw128(bo), 1);
        } else {
            Wgmma<N>::rs(d, h, desc_sw128(bo), acc);
        }
    }
}

// Tile geometry (identical in every role).  A tile is RT rays x SP = 64/RT consecutive samples: row = sub * RT +
// ray_in, so neighbouring rows are adjacent rays at the SAME sample index -- their volume / image taps fall in the
// same few cache lines.  Ray and sample of row `row` of tile `tile` of ray group `grp`:
struct TileRow {
    int ray, s_idx;
    bool valid;
    size_t si;
    __device__ __forceinline__ TileRow(const RenderIO& io, int grp, int tile, int row) {
        const int RT = io.rays_per_tile, SP = wg::ROWS / RT, rt_shift = 31 - __clz(RT);
        ray = grp * RT + (row & (RT - 1));
        s_idx = tile * SP + (row >> rt_shift);
        valid = ray < io.N && s_idx < io.S;
        si = (size_t)ray * io.S + s_idx;
    }
};

// Front end of one sample row: the operand columns the consumers' K-steps read.
//   PE   cols 0..31  = [x y z | sin(2^k x), first 29 of 30]          cols 32..63 = [sin(512 z) | cos(2^k x) | 0]
//   MISC cols 0..7   = volume features, 8..19 = colour (3 views x (r, g, b, mask)), 20..31 = 0,
//        cols 32..34 = view direction, 35..47 = 0
// Two threads per row (part 0 / 1).  fp16 (the producer warpgroup): part 0 takes the volume tap, the view direction
// and the sines, part 1 the three colour taps and the cosines -- even shares.  Split (each MMA warpgroup runs its own
// front end): part 0 only the sines, part 1 every gather and the cosines.
template <bool SPLIT>
__device__ __forceinline__ void store_pe_sin(uint8_t* pe, int row, const float* nd) {
    float v[32];
    v[0] = nd[0]; v[1] = nd[1]; v[2] = nd[2];
    float f = 1.f;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
            if (3 + 3 * k + j < 32) v[3 + 3 * k + j] = SPLIT ? sinf(nd[j] * f) : __sinf(nd[j] * f);
        f *= 2.f;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) store8<SPLIT>(pe, row, c, v + 8 * c);
}
template <bool SPLIT>
__device__ __forceinline__ void store_pe_cos(uint8_t* pe, int row, const float* nd) {
    float v[32];
    v[0] = SPLIT ? sinf(nd[2] * 512.f) : __sinf(nd[2] * 512.f);
    float f = 1.f;
#pragma unroll
    for (int k = 0; k < 10; ++k) {
#pragma unroll
        for (int j = 0; j < 3; ++j) v[1 + 3 * k + j] = SPLIT ? cosf(nd[j] * f) : __cosf(nd[j] * f);
        f *= 2.f;
    }
    v[31] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) store8<SPLIT>(pe, row, 4 + c, v + 8 * c);
}
// MISC cols 0..7 (volume), 24..31 (zero), 32..39 (view direction), 40..47 (zero); input_feat[0..7]
// VT: the volume's storage type (float, or __half for an fp16 volume)
template <bool SPLIT, typename VT>
__device__ __forceinline__ void store_volume_dir(const SceneDev& sc, const Cams& cams, const RenderIO& io, const TileRow& r,
                                                 const float* nd, float dx, float dy, float dz, uint8_t* misc, int row) {
    float feat[8], dir[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) feat[i] = 0.f;
    if (r.valid) {
        view_dir<SPLIT>(cams, dx, dy, dz, dir);
        sample_volume<VT>(sc, nd[0], nd[1], nd[2], feat);
        if (io.input_feat) {
            float4* o = reinterpret_cast<float4*>(io.input_feat + r.si * 20);
            o[0] = make_float4(feat[0], feat[1], feat[2], feat[3]);
            o[1] = make_float4(feat[4], feat[5], feat[6], feat[7]);
        }
    }
    const float z8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const float d8[8] = {dir[0], dir[1], dir[2], 0.f, 0.f, 0.f, 0.f, 0.f};
    store8<SPLIT>(misc, row, 0, feat);
    store8<SPLIT>(misc, row, 3, z8);
    store8<SPLIT>(misc, row, 4, d8);
    store8<SPLIT>(misc, row, 5, z8);
}
// MISC cols 8..23 (colour, then four zero columns); input_feat[8..19]
template <bool SPLIT>
__device__ __forceinline__ void store_color(const SceneDev& sc, const Cams& cams, const RenderIO& io, const TileRow& r,
                                            float px, float py, float pz, uint8_t* misc, int row) {
    float feat[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) feat[i] = 0.f;
    if (r.valid) {
#pragma unroll
        for (int vw = 0; vw < 3; ++vw) sample_color<SPLIT>(sc, cams, vw, px, py, pz, feat + 4 * vw);
        if (io.input_feat) {
            float4* o = reinterpret_cast<float4*>(io.input_feat + r.si * 20);
#pragma unroll
            for (int i = 0; i < 3; ++i) o[2 + i] = make_float4(feat[4 * i], feat[4 * i + 1], feat[4 * i + 2], feat[4 * i + 3]);
        }
    }
    store8<SPLIT>(misc, row, 1, feat);
    store8<SPLIT>(misc, row, 2, feat + 8);
}
template <bool FAST, bool SPLIT, typename VT>
__device__ __forceinline__ void front_end(const SceneDev& sc, const Cams& cams, const RenderIO& io, int grp, int tile,
                                          int t, uint8_t* pe, uint8_t* misc) {
    const int row = t & (wg::ROWS - 1), part = t >> 6;
    const TileRow r(io, grp, tile, row);
    float nx = 0.f, ny = 0.f, nz = 0.f;
    float px = 0.f, py = 0.f, pz = 0.f, dx = 0.f, dy = 0.f, dz = 1.f, z;      // z: the compositing recomputes it
    if (r.valid) sample_point<FAST, SPLIT>(sc, cams, io, r.ray, r.s_idx, r.si, px, py, pz, dx, dy, dz, nx, ny, nz, z);
    const float nd[3] = {nx, ny, nz};
    if (part == 0) {
        if (!SPLIT) store_volume_dir<SPLIT, VT>(sc, cams, io, r, nd, dx, dy, dz, misc, row);
        store_pe_sin<SPLIT>(pe, row, nd);
    } else {
        if (SPLIT) store_volume_dir<SPLIT, VT>(sc, cams, io, r, nd, dx, dy, dz, misc, row);
        store_color<SPLIT>(sc, cams, io, r, px, py, pz, misc, row);
        store_pe_cos<SPLIT>(pe, row, nd);
    }
}

// STOP: the state a consumer carries from pass to pass -- the verdict of the tile composited last (warp 0: every valid
// ray of the group has cT < t_stop), no work left, the current tile is its group's last, the current tile is its
// group's first (the previous one was a group's last), tiles computed
template <bool STOP> struct StopRegs { bool verdict = false, idle = false, last = false, first = true; uint32_t ncomp = 0; };
template <> struct StopRegs<false> { static constexpr bool last = false; };

// STOP (early ray termination; the ray entry, FAST, and the samples entry): after compositing tile k of a group, if every valid ray of the group has
// transmittance cT < t_stop, the group's tiles k + 3 onwards are not computed (k + 1 and k + 2 are composited as
// usual), and the number of passes of a CTA becomes dynamic.  Each consumer computes its plan for pass p + 2 at the
// start of pass p: the next tile of its group, or the next group of the CTA's list (a shared counter, in order of
// demand), or idle.  Tile k + 2 depends only on the verdicts up to tile k - 1, so every plan is known two passes ahead
// and the producer fills a slot as soon as its consumer releases it, as without STOP.  Without STOP the kernel is the
// one it always was (t_stop, tiles_done and ranges are unused).
// STOP with a range table (empty-space skipping, from occ_ranges_kernel): group g is computed over its tiles
// [ranges[g].x, ranges[g].y] only -- its first plan starts at .x, its last tile is .y, the t_stop rule counts computed
// tiles -- and a group with an empty range is not handed out (the pre-pass stored its pixels).  Null: [0, NT - 1].
// Only the STOP instantiations take the table (Table = const int2*, read through range_table inside STOP code): the
// others keep their five parameters, because one more kernel parameter alone changes the split kernels' register
// allocation.
// VT = __half: the encoding volume is stored as fp16 (sc.vol points at halves); only the volume gather changes.
template <bool FAST, bool SPLIT, bool STOP = false, typename VT = float, typename... Table>
__global__ void __launch_bounds__(wg::threads(SPLIT, !SPLIT && !STOP), 1)
render_wg_kernel(const SceneDev sc, const RenderIO io, const uint8_t* __restrict__ wimg, float t_stop,
                 unsigned long long* tiles_done, Table... table) {
    using namespace wg;
    constexpr bool RMOD = !SPLIT && !STOP;               // the modulation in the consumers' registers
    constexpr int NS = nstage(SPLIT, RMOD), THREADS = threads(SPLIT, RMOD);
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ std::conditional_t<RMOD, WgSharedRes, WgShared<SPLIT>> sh;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float* bias = reinterpret_cast<float*>(smem + off_bias(SPLIT, RMOD));

    load_cams(sc, &sh.cams, tid);
    for (int i = tid; i < BIAS_FLOATS; i += THREADS) bias[i] = __ldg(reinterpret_cast<const float*>(wimg + tail_offset(SPLIT)) + i);
    if (tid == 0) {
        for (int i = 0; i < NS; ++i) { mbar_init(&sh.full[i], 1); mbar_init(&sh.empty[i], NWG * 4); }
        if (!SPLIT)
            for (int i = 0; i < SLOTS; ++i) { mbar_init(&sh.slot_full[i], 128); mbar_init(&sh.slot_empty[i], 4); }
        if constexpr (RMOD) mbar_init(&sh.resident, 1);
        if constexpr (STOP) {
            WgStop* ss = stop_state(smem, SPLIT);
            const int G0 = (io.N + io.rays_per_tile - 1) / io.rays_per_tile;
            const int NT0 = (io.S + wg::ROWS / io.rays_per_tile - 1) / (wg::ROWS / io.rays_per_tile);
            for (int i = 0; i < STOP_SLOTS; ++i) mbar_init(&ss->dec[i], NWG);
            const int2* ranges = range_table(table...);
            int next = 0;                               // passes 0 and 1: first groups, then their next tile (or the next group)
            auto take = [&]() { return next++; };
            for (int w = 0; w < NWG; ++w) {
                const int2 p0 = stop_take(ranges, take, G0, NT0);
                int2 p1 = make_int2(-1, 0);
                if (p0.x >= 0)
                    p1 = p0.y + 1 <= stop_range(ranges, p0.x, NT0).y ? make_int2(p0.x, p0.y + 1) : stop_take(ranges, take, G0, NT0);
                ss->plan[0][w] = p0;
                ss->plan[1][w] = p1;
            }
            ss->next = next;
        }
        fence_barrier_init();
    }
    __syncthreads();

    // ---- work decomposition (identical in every role) ---------------------------------------------
    // Warpgroup (consumer) w walks the NT tiles of its RT-ray group front to back; the compositing state is carried
    // in registers.  Any S works.
    const int N = io.N, S = io.S;
    const int RT = io.rays_per_tile, SP = ROWS / RT;
    const int NT = (S + SP - 1) / SP;
    const int G = (N + RT - 1) / RT;
    const int units_total = (G + NWG - 1) / NWG;
    const int my_units = blockIdx.x < units_total ? (units_total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const int npass = my_units * NT;
    const uint32_t ring = smem_u32(smem + off_ring(SPLIT, RMOD));
    auto group_of = [&](int pass, int w) { return ((pass / NT) * (int)gridDim.x + (int)blockIdx.x) * NWG + w; };

    // RMOD: each role sets its register budget first thing in its own branch (the loader and the producer give theirs
    // up to the consumers), so that ptxas allocates every role's code within that role's budget
    if (SPLIT ? warp == loader_warp(true) : warp >= loader_warp(false)) {
        // =========================== weight loader ===================================================
        // RMOD: the first warp of the loader warpgroup; the other three leave
        if constexpr (RMOD) setmaxnreg_dec<REGS_LOADER>();
        if ((SPLIT || warp == loader_warp(false)) && elect_one()) {
            uint32_t n = 0;
            if constexpr (RMOD) {                        // the resident chunks once, then only the streamed ones
                mbar_arrive_expect_tx(&sh.resident, RES_BYTES);
#pragma unroll
                for (int c = 0; c < NCHUNK; ++c)
                    if (resident(c))
                        bulk_load(smem + off_res() + res_offset(c), wimg + (size_t)c * HALF_STRIDE, chunk_rows(c) * 128, &sh.resident);
#pragma unroll 1
                for (int pass = 0; pass < npass; ++pass) {
#pragma unroll 1
                    for (int c = 0; c < NCHUNK; ++c) {
                        if (resident(c)) continue;
                        const uint32_t st = n % NS;
                        if (n >= (uint32_t)NS) mbar_wait(&sh.empty[st], ((n / NS) - 1) & 1);
                        const uint32_t bytes = (uint32_t)chunk_rows(c) * 128;
                        mbar_arrive_expect_tx(&sh.full[st], bytes);
                        bulk_load(smem + off_ring(false, true) + st * HALF_STRIDE, wimg + (size_t)c * HALF_STRIDE, bytes, &sh.full[st]);
                        ++n;
                    }
                }
            } else {
#pragma unroll 1
                for (int pass = 0; STOP || pass < npass; ++pass) {
                    if constexpr (STOP) {                    // one pass of NCHUNK chunks while any consumer has work
                        WgStop* ss = stop_state(smem, SPLIT);
                        stop_wait(ss, pass);
                        bool any = false;
#pragma unroll
                        for (int w = 0; w < NWG; ++w) any |= stop_busy(ss, pass, w);
                        if (!any) break;
                    }
#pragma unroll 1
                    for (int c = 0; c < NCHUNK; ++c, ++n) {
                        const uint32_t st = n % NS;
                        if (n >= (uint32_t)NS) mbar_wait(&sh.empty[st], ((n / NS) - 1) & 1);
                        const uint32_t bytes = (uint32_t)chunk_rows(c) * 128;
                        uint8_t* dst = smem + off_ring(SPLIT, RMOD) + st * chunk_stride(SPLIT);
                        const uint8_t* src = wimg + (size_t)c * chunk_stride(SPLIT);
                        mbar_arrive_expect_tx(&sh.full[st], SPLIT ? 2 * bytes : bytes);
                        bulk_load(dst, src, bytes, &sh.full[st]);
                        if (SPLIT) bulk_load(dst + HALF_STRIDE, src + HALF_STRIDE, bytes, &sh.full[st]);
                    }
                }
            }
        }
        return;
    }
    if constexpr (!SPLIT) {
        if (warp >= NWG * 4) {
            // ======================= producer: front ends of the consumers' tiles, in their order ============
            // consumer w's k-th tile goes to slot 2 w + (k & 1)
            if constexpr (RMOD) setmaxnreg_dec<REGS_PRODUCER>();
            const int t = tid & 127;
            uint32_t filled[NWG];
#pragma unroll
            for (int w = 0; w < NWG; ++w) filled[w] = 0;
#pragma unroll 1
            for (int pass = 0; STOP || pass < npass; ++pass) {
                int2 pl[NWG];                            // STOP: the consumers' plans for this pass
                if constexpr (STOP) {
                    WgStop* ss = stop_state(smem, SPLIT);
                    stop_wait(ss, pass);
                    bool any = false;
#pragma unroll
                    for (int w = 0; w < NWG; ++w) { pl[w] = stop_plan(ss, pass, w); any |= pl[w].x >= 0; }
                    if (!any) break;
                }
#pragma unroll
                for (int w = 0; w < NWG; ++w) {
                    const int grp = STOP ? pl[w].x : group_of(pass, w);
                    if (STOP ? grp < 0 : grp >= G) continue;
                    const int s = 2 * w + (filled[w] & 1);
                    if (filled[w] >= 2) mbar_wait(&sh.slot_empty[s], ((filled[w] >> 1) - 1) & 1);
                    uint8_t* pe = smem + s * SLOT_BYTES;
                    front_end<FAST, false, VT>(sc, sh.cams, io, grp, STOP ? pl[w].y : pass % NT, t, pe, pe + tile_bytes(false));
                    fence_proxy_async();
                    mbar_arrive(&sh.slot_full[s]);
                    ++filled[w];
                }
            }
            return;
        }
        if constexpr (RMOD) {
            setmaxnreg_inc<REGS_CONSUMER>();
            mbar_wait(&sh.resident, 0);                  // the resident chunks have landed
        }
    }

    // =========================== MMA warpgroups: one tile at a time ====================================
    const int wgi = warp >> 2, t = tid & 127, w4 = (tid >> 5) & 3, g = lane >> 2, q = lane & 3;
    uint8_t* state = smem + off_state(SPLIT, RMOD, wgi);
    float* modp = reinterpret_cast<float*>(state) + t;                              // !RMOD: [i][128 threads]
    float* xch = reinterpret_cast<float*>(state + (RMOD ? 0 : MOD_BYTES));          // [64 rows][alpha, r, g, b]
    const int row_a = w4 * 16 + g, row_b = row_a + 8;
    uint32_t nchunk = 0, ntile = 0;
    // the k-th streamed chunk after the oldest one not yet released (k > 0: RMOD only)
    auto acquire = [&](uint32_t k = 0) -> uint32_t {
        const uint32_t st = (nchunk + k) % NS;
        mbar_wait(&sh.full[st], ((nchunk + k) / NS) & 1);
        return ring + st * chunk_stride(SPLIT);
    };
    auto release = [&]() {
        __syncwarp();
        if (lane == 0) mbar_arrive(&sh.empty[nchunk % NS]);
        ++nchunk;
    };
    // A layer of chunks c0 .. c0 + n - 1: layer_begin(c0, b[n]); per chunk i: chunk_begin(b[i]), wgmma_fence(), its
    // wgmmas, chunk_end(c0 + i, i == 0, d); then layer_end(c0 + n - 1, d).  Without RMOD every chunk is streamed,
    // acquired and drained on its own.  RMOD: layer_begin takes the B operands of the whole layer before its first wgmma
    // -- a resident chunk's is a constant address, a streamed one's waits for its stage -- and the layer's wgmma groups
    // stay in flight until one wait before its epilogue.  A streamed stage is released once the group that read it has
    // retired: wgmma_wait<1> after the layer's next group, or the layer's wait.
    const uint32_t res = ring + (off_res() - off_ring(false, true));
    auto layer_begin = [&](int c0, auto& b) {
        if constexpr (RMOD) {
            uint32_t k = 0;                              // the layer's streamed chunks taken so far
#pragma unroll
            for (int i = 0; i < (int)(sizeof(b) / sizeof(b[0])); ++i)
                b[i] = resident(c0 + i) ? res + res_offset(c0 + i) : acquire(k++);
        }
    };
    auto chunk_begin = [&](uint32_t b) -> uint32_t {
        if constexpr (RMOD) return b;
        else return acquire();
    };
    auto chunk_end = [&](int c, bool first, auto& d) {
        wgmma_commit();
        if constexpr (!RMOD) {
            wgmma_wait<0>(); reg_fence(d);
            release();
        } else if (!first && !resident(c - 1)) {
            wgmma_wait<1>(); release();
        }
    };
    auto layer_end = [&](int c, auto& d) {
        if constexpr (RMOD) {
            wgmma_wait<0>(); reg_fence(d);
            if (!resident(c)) release();
        }
    };
    auto col_of = [&](int i) { return 8 * (i >> 2) + 2 * q + (i & 1); };

    float cT = 1.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f, c4 = 0.f;   // compositing state of ray t (t < RT)
    float acc[64];
    uint32_t ah[32], al[SPLIT ? 32 : 1];
    float mod[RMOD ? 64 : 1];                           // RMOD: the modulation of the current tile, accumulator layout
    auto mod_of = [&](int i) -> float {
        if constexpr (RMOD) return mod[i];
        else return modp[i * 128];
    };
    // fp16: the bias pair of columns 8 j + 2 q, 8 j + 2 q + 1 (both rows of a thread use it: one 8-byte load)
    auto bias2 = [&](int base, int j) { return *reinterpret_cast<const float2*>(bias + base + 8 * j + 2 * q); };
    // split: 2^-ew, the scale of the register activation rows row_a / row_b, and the factor that takes the current
    // accumulator rows back to their true values (fp16: all 1)
    const float inv_w = SPLIT ? bias[BIAS_WINV] : 1.f;
    float sa = 1.f, sb = 1.f, ia = inv_w, ib = inv_w;

    StopRegs<STOP> sr;

#pragma unroll 1
    for (int pass = 0; STOP || pass < npass; ++pass) {
        int grp = group_of(pass, wgi), tile = pass % NT;
        if constexpr (STOP) {
            WgStop* ss = stop_state(smem, SPLIT);
            if (!sr.idle) {                              // own plans: written by thread 0 before named barriers
                const int2 pl = stop_plan(ss, pass, wgi);
                grp = pl.x; tile = pl.y; sr.idle = grp < 0;
            }
            if (sr.idle) {                                  // keep the weight ring moving while another consumer works
                stop_wait(ss, pass);
                bool any = false;
#pragma unroll
                for (int w = 0; w < NWG; ++w) any |= w != wgi && stop_busy(ss, pass, w);
                if (!any) break;
                if (t == 0) {
                    ss->plan[(pass + 2) & (STOP_SLOTS - 1)][wgi] = make_int2(-1, 0);
                    mbar_arrive(&ss->dec[(pass + 2) & (STOP_SLOTS - 1)]);
                }
#pragma unroll 1
                for (int c = 0; c < NCHUNK; ++c) { acquire(); release(); }
                continue;
            }
            // from the plan of pass + 1, (g, k): tile k + 1 of g is skipped iff k is the last of g's range (NT - 1 without
            // a range table) or the verdict of tile k - 2 (this consumer's last composited tile, if it is one of g's)
            // says stop
            if (t == 0) {
                const int2 p1 = stop_plan(ss, pass + 1, wgi);
                int2 nx = make_int2(-1, 0);
                if (p1.x >= 0) {
                    const int2* ranges = range_table(table...);
                    const int2 r = stop_range(ranges, p1.x, NT);
                    nx = make_int2(p1.x, p1.y + 1);
                    if (p1.y + 1 > r.y || (p1.y >= r.x + 2 && sr.verdict))
                        nx = stop_take(ranges, [&]() { return atomicAdd(&ss->next, 1); }, G, NT);
                }
                ss->plan[(pass + 2) & (STOP_SLOTS - 1)][wgi] = nx;
                mbar_arrive(&ss->dec[(pass + 2) & (STOP_SLOTS - 1)]);
            }
            ++sr.ncomp;
        } else {
            if (grp >= G) {                              // idle in the final passes: keep the weight ring moving
#pragma unroll 1
                for (int c = 0; c < (RMOD ? NSTREAM : NCHUNK); ++c) { acquire(); release(); }
                continue;
            }
        }
        uint32_t pe_u, misc_u, slot = 0;
        named_bar_sync(1 + wgi, 128);                    // the previous tile's exchange (split: operand tiles) is consumed
        if constexpr (SPLIT) {
            // -------------------------- front end (split mode: this warpgroup's own operand tiles) -------------
            uint8_t* pe = smem + wgi * wg_bytes(true);
            uint8_t* misc = pe + off_misc(true);
            front_end<FAST, true, VT>(sc, sh.cams, io, grp, tile, t, pe, misc);
            fence_proxy_async();
            named_bar_sync(1 + wgi, 128);
            pe_u = smem_u32(pe); misc_u = smem_u32(misc);
        } else {
            // -------------------------- operand tiles from the producer -----------------------------------
            slot = 2 * wgi + (ntile & 1);
            mbar_wait(&sh.slot_full[slot], (ntile >> 1) & 1);
            ++ntile;
            pe_u = smem_u32(smem + slot * SLOT_BYTES); misc_u = pe_u + tile_bytes(false);
        }

        // -------------------------- modulation: pts_bias(features), K = 20 -> registers (RMOD) or shared memory
        {
            uint32_t bl[1];
            layer_begin(0, bl);
            const uint32_t b = chunk_begin(bl[0]);
            wgmma_fence();
            gemm_ss<128, SPLIT>(acc, misc_u, b, 0, 2, true);
            chunk_end(0, true, acc); layer_end(0, acc);
            if constexpr (!RMOD) {
#pragma unroll
                for (int i = 0; i < 64; ++i) modp[i * 128] = fmaf(acc[i], inv_w, bias[BIAS_MOD + col_of(i)]);
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const float2 bm = bias2(BIAS_MOD, j);
                    mod[4 * j + 0] = fmaf(acc[4 * j + 0], inv_w, bm.x);
                    mod[4 * j + 1] = fmaf(acc[4 * j + 1], inv_w, bm.y);
                    mod[4 * j + 2] = fmaf(acc[4 * j + 2], inv_w, bm.x);
                    mod[4 * j + 3] = fmaf(acc[4 * j + 3], inv_w, bm.y);
                }
            }
        }
        // -------------------------- trunk: six layers, h = relu((W x + b) * mod) -----------------------------
        auto trunk_epilogue = [&](int l) {
            if constexpr (SPLIT) {
#pragma unroll
                for (int i = 0; i < 64; ++i)
                    acc[i] = fmaxf(fmaf(acc[i], (i & 2) ? ib : ia, bias[BIAS_TRUNK + l * 128 + col_of(i)]) * modp[i * 128], 0.f);
                split_rows<64>(acc, ah, al, sa, sb);
                ia = inv_pow2(sa) * inv_w; ib = inv_pow2(sb) * inv_w;
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const float2 bt = bias2(BIAS_TRUNK + l * 128, j);
#pragma unroll
                    for (int i = 4 * j; i < 4 * j + 4; i += 2) {
                        float v0 = (acc[i] + bt.x) * mod_of(i);
                        float v1 = (acc[i + 1] + bt.y) * mod_of(i + 1);
                        v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
                        ah[i >> 1] = cvt_h2_sat(v0, v1);
                    }
                }
            }
        };
        {   // layer 0: A = encoding (63 columns)
            uint32_t bl[1];
            layer_begin(1, bl);
            const uint32_t b = chunk_begin(bl[0]);
            wgmma_fence();
            gemm_ss<128, SPLIT>(acc, pe_u, b, 0, 4, true);
            chunk_end(1, true, acc); layer_end(1, acc);
            ia = ib = inv_w;
            trunk_epilogue(0);
        }
#pragma unroll 1
        for (int l = 1; l <= 4; ++l) {
            uint32_t bl[2];
            layer_begin(2 * l, bl);
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
                const uint32_t b = chunk_begin(bl[kb]);
                wgmma_fence();
                gemm_rs<128, SPLIT>(acc, ah, al, b, kb, kb == 0);
                chunk_end(2 * l + kb, kb == 0, acc);
            }
            layer_end(2 * l + 1, acc);
            trunk_epilogue(l);
        }
        {   // layer 5: A = [encoding | h] (skip connection after layer 4)
            uint32_t bl[3];
            layer_begin(10, bl);
            uint32_t b = chunk_begin(bl[0]);
            wgmma_fence();
            gemm_ss<128, SPLIT>(acc, pe_u, b, 0, 4, true);
            chunk_end(10, true, acc);
            if constexpr (SPLIT) {                     // to the scale of the register rows (exact: powers of two)
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[i] *= (i & 2) ? sb : sa;
            }
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
                b = chunk_begin(bl[1 + kb]);
                wgmma_fence();
                gemm_rs<128, SPLIT>(acc, ah, al, b, kb, false);
                chunk_end(11 + kb, false, acc);
            }
            layer_end(12, acc);
            trunk_epilogue(5);
        }
        // -------------------------- folded head: views layer (64) + alpha (col 64) ---------------------------
        float sig_a = 0.f, sig_b = 0.f;
        {
            float h72[36];
            uint32_t bl[3];
            layer_begin(13, bl);
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
                const uint32_t b = chunk_begin(bl[kb]);
                wgmma_fence();
                gemm_rs<72, SPLIT>(h72, ah, al, b, kb, kb == 0);
                chunk_end(13 + kb, kb == 0, h72);
            }
            if constexpr (SPLIT) {                     // back to the front-end scale of the view-direction columns
                const float ra = inv_pow2(sa), rb = inv_pow2(sb);
#pragma unroll
                for (int i = 0; i < 36; ++i) h72[i] *= (i & 2) ? rb : ra;
            }
            {   // view direction: MISC K-step 2 (cols 32..47)
                const uint32_t b = chunk_begin(bl[2]);
                wgmma_fence();
                gemm_ss<72, SPLIT>(h72, misc_u, b, 2, 1, false);
                chunk_end(15, false, h72); layer_end(15, h72);
                if constexpr (!SPLIT) {                // the last read of the operand tiles: free the slot
                    if (lane == 0) mbar_arrive(&sh.slot_empty[slot]);
                }
            }
            if constexpr (SPLIT) {
#pragma unroll
                for (int i = 0; i < 32; ++i) h72[i] = fmaxf(fmaf(h72[i], inv_w, bias[BIAS_HEAD + col_of(i)]), 0.f);
                split_rows<32>(h72, ah, al, sa, sb);
                ia = inv_pow2(sa) * inv_w; ib = inv_pow2(sb) * inv_w;
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float2 bh = bias2(BIAS_HEAD, j);
#pragma unroll
                    for (int i = 4 * j; i < 4 * j + 4; i += 2) {
                        const float v0 = fmaxf(h72[i] + bh.x, 0.f);
                        const float v1 = fmaxf(h72[i + 1] + bh.y, 0.f);
                        ah[i >> 1] = cvt_h2_sat(v0, v1);
                    }
                }
            }
            sig_a = fmaxf(fmaf(h72[32], inv_w, bias[BIAS_HEAD + 64]), 0.f);
            sig_b = fmaxf(fmaf(h72[34], inv_w, bias[BIAS_HEAD + 64]), 0.f);
        }
        // -------------------------- rgb (N = 8, 3 used) -------------------------------------------------------
        {
            float r8[4];
            uint32_t bl[1];
            layer_begin(16, bl);
            const uint32_t b = chunk_begin(bl[0]);
            wgmma_fence();
            gemm_rs<8, SPLIT>(r8, ah, al, b, 0, true);
            chunk_end(16, true, r8); layer_end(16, r8);
            auto sigm = [&](float x) { return SPLIT ? __fdiv_rn(1.f, 1.f + expf(-x)) : __fdividef(1.f, 1.f + __expf(-x)); };
            if (q == 0) {
                xch[row_a * 4 + 0] = 1.f - (SPLIT ? expf(-sig_a) : __expf(-sig_a));
                xch[row_b * 4 + 0] = 1.f - (SPLIT ? expf(-sig_b) : __expf(-sig_b));
                xch[row_a * 4 + 1] = sigm(fmaf(r8[0], ia, bias[BIAS_RGB + 0]));
                xch[row_a * 4 + 2] = sigm(fmaf(r8[1], ia, bias[BIAS_RGB + 1]));
                xch[row_b * 4 + 1] = sigm(fmaf(r8[2], ib, bias[BIAS_RGB + 0]));
                xch[row_b * 4 + 2] = sigm(fmaf(r8[3], ib, bias[BIAS_RGB + 1]));
            } else if (q == 1) {
                xch[row_a * 4 + 3] = sigm(fmaf(r8[0], ia, bias[BIAS_RGB + 2]));
                xch[row_b * 4 + 3] = sigm(fmaf(r8[2], ib, bias[BIAS_RGB + 2]));
            }
        }
        named_bar_sync(1 + wgi, 128);
        if constexpr (STOP) {                            // the group's last tile unless pass + 1 plans (grp, tile + 1)
            const int2 p1 = stop_plan(stop_state(smem, SPLIT), pass + 1, wgi);
            sr.last = !(p1.x == grp && p1.y == tile + 1);
        }
        // -------------------------- compositing (renderer.py:18-26,65-92) ----------------------------------
        // the first RT threads walk their ray's SP samples of this tile front to back -- the reference's
        // sequential cumprod order
        if (t < RT) {
            if constexpr (STOP) {                        // the group's first tile: the first of its range
                if (sr.first) { cT = 1.f; c0 = c1 = c2 = c3 = c4 = 0.f; }
            } else {
                if (tile == 0) { cT = 1.f; c0 = c1 = c2 = c3 = c4 = 0.f; }
            }
            const int cray = grp * RT + t;
            if (cray < N) {
                float znear = 0.f, zfar = 0.f;
                if (FAST) { const float4 r1 = __ldg(reinterpret_cast<const float4*>(io.rays + (size_t)cray * 8) + 1); znear = r1.z; zfar = r1.w; }
                for (int sub = 0; sub < SP; ++sub) {
                    const int sj = tile * SP + sub;
                    if (sj >= S) break;
                    const float4 v = reinterpret_cast<const float4*>(xch)[sub * RT + t];
                    float z;
                    if (FAST) z = ray_z(znear, zfar, __ldg(io.t_steps + sj), io.rg.lindisp);
                    else      z = __ldg(io.z + (size_t)cray * S + sj);
                    const float wgt = v.x * cT;
                    if (io.alpha) io.alpha[(size_t)cray * S + sj] = v.x;
                    if (io.weights) io.weights[(size_t)cray * S + sj] = wgt;
                    c0 = fmaf(wgt, v.y, c0); c1 = fmaf(wgt, v.z, c1); c2 = fmaf(wgt, v.w, c2);
                    c3 = fmaf(wgt, z, c3); c4 += wgt;
                    cT *= (1.f - v.x) + 1e-10f;
                }
                if (STOP ? sr.last : tile == NT - 1) {
                    float o0 = c0, o1 = c1, o2 = c2;
                    if (sc.white_bkgd) { const float bg = 1.f - c4; o0 += bg; o1 += bg; o2 += bg; }
                    store_pixel(io, cray, o0, o1, o2, c3);
                }
            }
        }
        if constexpr (STOP) {                            // rays past the batch end (and lanes >= RT) count as stopped
            if (t < 32) sr.verdict = __all_sync(0xffffffffu, t >= RT || grp * RT + t >= N || cT < t_stop);
            sr.first = sr.last;
        }
    }
    if constexpr (STOP) {
        if (t == 0 && tiles_done) atomicAdd(tiles_done, (unsigned long long)sr.ncomp);
    }
}

// the dynamic shared memory of the eight instantiations with volume storage VT
template <typename VT>
static int set_wg_smem_attributes() {
    using namespace wg;
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<true, false, false, VT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(false, true)));
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<false, false, false, VT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(false, true)));
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<true, true, false, VT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(true, false)));
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<false, true, false, VT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(true, false)));
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<true, false, true, VT, const int2*>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(false, false) + STOP_BYTES));
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<true, true, true, VT, const int2*>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(true, false) + STOP_BYTES));
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<false, false, true, VT, const int2*>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(false, false) + STOP_BYTES));
    MVSN_CUDA_CHECK(cudaFuncSetAttribute(render_wg_kernel<false, true, true, VT, const int2*>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(true, false) + STOP_BYTES));
    return MVSN_OK;
}

template <typename VT>
static void launch_wg_kernel(int grid, cudaStream_t stream, const SceneDev& sc, const RenderIO& io, const uint8_t* w, bool fast,
                             bool split, const float* t_stop, unsigned long long* tiles_done, const int2* ranges) {
    using namespace wg;
    if (t_stop) {                                         // early ray termination: the ray and the samples entries
        const int smem = smem_bytes(split, false) + STOP_BYTES, nthreads = threads(split, false);
        if (fast) {
            if (split) render_wg_kernel<true, true, true, VT, const int2*><<<grid, nthreads, smem, stream>>>(sc, io, w, *t_stop, tiles_done, ranges);
            else       render_wg_kernel<true, false, true, VT, const int2*><<<grid, nthreads, smem, stream>>>(sc, io, w, *t_stop, tiles_done, ranges);
        } else {
            if (split) render_wg_kernel<false, true, true, VT, const int2*><<<grid, nthreads, smem, stream>>>(sc, io, w, *t_stop, tiles_done, ranges);
            else       render_wg_kernel<false, false, true, VT, const int2*><<<grid, nthreads, smem, stream>>>(sc, io, w, *t_stop, tiles_done, ranges);
        }
    } else if (split) {
        const int smem = smem_bytes(true, false), nthreads = threads(true, false);
        if (fast) render_wg_kernel<true, true, false, VT><<<grid, nthreads, smem, stream>>>(sc, io, w, 0.f, nullptr);
        else      render_wg_kernel<false, true, false, VT><<<grid, nthreads, smem, stream>>>(sc, io, w, 0.f, nullptr);
    } else {
        const int smem = smem_bytes(false, true), nthreads = threads(false, true);
        if (fast) render_wg_kernel<true, false, false, VT><<<grid, nthreads, smem, stream>>>(sc, io, w, 0.f, nullptr);
        else      render_wg_kernel<false, false, false, VT><<<grid, nthreads, smem, stream>>>(sc, io, w, 0.f, nullptr);
    }
}

int launch_render_wg(const SceneDev& sc, const RenderIO& io_in, bool fast, bool split, const void* wimg, cudaStream_t stream,
                     const float* t_stop, unsigned long long* tiles_done, bool half_vol, const uint32_t* occ_bits,
                     int2* ranges) {
    using namespace wg;
    RenderIO io = io_in;
    static bool attr_set[64] = {false};                   // once per device, not per launch
    int dev = 0;
    MVSN_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !attr_set[dev]) {
        int rc = set_wg_smem_attributes<float>();
        if (rc) return rc;
        if ((rc = set_wg_smem_attributes<__half>())) return rc;
        if (dev < 64) attr_set[dev] = true;
    }
    // rays per tile: 32 (best gather locality) unless the batch is too small to give every warpgroup a group
    int rt = 32;
    while (rt > 4 && (io.N + rt - 1) / rt < NWG * sm_count()) rt >>= 1;
    io.rays_per_tile = rt;
    const int G = (io.N + rt - 1) / rt;
    const int units = (G + NWG - 1) / NWG;
    const int grid = units < sm_count() ? units : sm_count();
    if (grid <= 0) return MVSN_OK;
    const uint8_t* w = static_cast<const uint8_t*>(wimg);
    if (occ_bits) {                                       // empty-space skipping: the range pre-pass at this launch's rt
        if (!t_stop || !ranges) { set_error("launch_render_wg: an occupancy grid needs t_stop and a range table"); return MVSN_EBADSHAPE; }
        const int rc = launch_occupancy_ranges(sc, io, split, occ_bits, ranges, stream);
        if (rc) return rc;
    } else {
        ranges = nullptr;
    }
    if (half_vol) launch_wg_kernel<__half>(grid, stream, sc, io, w, fast, split, t_stop, tiles_done, ranges);
    else          launch_wg_kernel<float>(grid, stream, sc, io, w, fast, split, t_stop, tiles_done, ranges);
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

// ------------------------------------------------------------------------------------------------
// fp16 volume image: [8][nvox] (planar) or [nvox][8] (channels-last), fp32 or fp16 -> [nvox][8] fp16, rounded as
// Tensor.half() rounds (__float2half_rn: overflow to inf, subnormals kept; an fp16 source is copied)
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void volume_to_half_kernel(const T* __restrict__ src, bool planar, long long nvox, uint4* __restrict__ dst) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvox; i += (long long)gridDim.x * blockDim.x) {
        __half h[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const T v = planar ? src[c * nvox + i] : src[8 * i + c];
            if constexpr (std::is_same<T, __half>::value) h[c] = v;
            else h[c] = __float2half_rn(v);
        }
        uint4 o;
        o.x = (uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16);
        o.y = (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16);
        o.z = (uint32_t)__half_as_ushort(h[4]) | ((uint32_t)__half_as_ushort(h[5]) << 16);
        o.w = (uint32_t)__half_as_ushort(h[6]) | ((uint32_t)__half_as_ushort(h[7]) << 16);
        dst[i] = o;
    }
}

int launch_volume_to_half(const void* src, bool src_half, bool src_planar, long long nvox, void* dst, cudaStream_t stream) {
    const int grid = cdiv(nvox, 256) < 8192 ? cdiv(nvox, 256) : 8192;
    if (src_half)
        volume_to_half_kernel<__half><<<grid, 256, 0, stream>>>(static_cast<const __half*>(src), src_planar, nvox, static_cast<uint4*>(dst));
    else
        volume_to_half_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const float*>(src), src_planar, nvox, static_cast<uint4*>(dst));
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

// ------------------------------------------------------------------------------------------------
// weight image packer (fp32 nn.Linear tensors -> fp16 (split: hi | lo, x2^ew) pre-swizzled chunks + fp32 biases)
// ------------------------------------------------------------------------------------------------
struct MlpPtrsWg { const float* p[MVSN_N_MLP_TENSORS]; };

// tensor indices: 0..11 pts_linears (w,b) x6; 12,13 pts_bias; 14,15 views; 16,17 feature; 18,19 alpha; 20,21 rgb
__device__ float wg_weight(const MlpPtrsWg& w, int c, int r, int k) {
    if (c == 0) return k < 20 ? w.p[12][r * 20 + k] : 0.f;
    if (c == 1) return k < 63 ? w.p[0][r * 63 + k] : 0.f;
    if (c <= 9) { const int l = c / 2, kb = c & 1; return w.p[2 * l][r * 128 + kb * 64 + k]; }
    if (c == 10) return k < 63 ? w.p[10][r * 191 + k] : 0.f;
    if (c <= 12) return w.p[10][r * 191 + 63 + (c - 11) * 64 + k];
    if (c <= 14) {                                 // views_linears[0][:, :128] @ feature_linear, then alpha_linear
        const int kk = (c - 13) * 64 + k;
        if (r < 64) {
            double s = 0.0;
            for (int j = 0; j < 128; ++j) s += (double)w.p[14][r * 131 + j] * (double)w.p[16][j * 128 + kk];
            return (float)s;
        }
        return r == 64 ? w.p[18][kk] : 0.f;
    }
    if (c == 15) return (r < 64 && k >= 32 && k < 35) ? w.p[14][r * 131 + 128 + (k - 32)] : 0.f;
    return r < 3 ? w.p[20][r * 64 + k] : 0.f;
}

// split mode: the largest |weight| of the image (its fp32 bits; atomicMax orders non-negative floats) -> tail[BIAS_WMAX],
// which the caller has zeroed
__global__ void wmax_mlp_wg_kernel(MlpPtrsWg w, uint8_t* __restrict__ out) {
    using namespace wg;
    const int c = blockIdx.x;
    float m = 0.f;
    for (int i = threadIdx.x; i < chunk_rows(c) * 64; i += blockDim.x) m = fmaxf(m, fabsf(wg_weight(w, c, i >> 6, i & 63)));
    atomicMax(reinterpret_cast<unsigned int*>(out + tail_offset(true)) + BIAS_WMAX, __float_as_uint(m));
}

__global__ void pack_mlp_wg_kernel(MlpPtrsWg w, bool split, uint8_t* __restrict__ out) {
    using namespace wg;
    const int c = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const float sw = split ? weight_scale(reinterpret_cast<const uint32_t*>(out + tail_offset(true))[BIAS_WMAX]) : 1.f;
    if (c == NCHUNK) {                             // fp32 bias tail
        float* b = reinterpret_cast<float*>(out + tail_offset(split));
        for (int i = tid; i < BIAS_FLOATS; i += nt) {
            if (split && i == BIAS_WMAX) continue;
            float v = 0.f;
            if (i < BIAS_TRUNK) v = w.p[13][i];
            else if (i < BIAS_HEAD) { const int l = (i - BIAS_TRUNK) / 128; v = w.p[2 * l + 1][(i - BIAS_TRUNK) % 128]; }
            else if (i < BIAS_HEAD + 64) {
                const int n = i - BIAS_HEAD;
                double s = (double)w.p[15][n];
                for (int j = 0; j < 128; ++j) s += (double)w.p[14][n * 131 + j] * (double)w.p[17][j];
                v = (float)s;
            } else if (i == BIAS_HEAD + 64) v = w.p[19][0];
            else if (i >= BIAS_RGB && i < BIAS_RGB + 3) v = w.p[21][i - BIAS_RGB];
            else if (split && i == BIAS_WINV) v = 1.f / sw;
            b[i] = v;
        }
        return;
    }
    uint8_t* dst = out + (size_t)c * chunk_stride(split);
    for (int i = tid * 16; i < chunk_stride(split); i += nt * 16) *reinterpret_cast<uint4*>(dst + i) = make_uint4(0, 0, 0, 0);
    __syncthreads();
    for (int i = tid; i < chunk_rows(c) * 64; i += nt) {
        const int r = i >> 6, k = i & 63;
        const uint32_t off = sw128_offset(r, k);
        const float v = wg_weight(w, c, r, k);
        if (split) {
            const __half h = __float2half_rn(v * sw);
            *reinterpret_cast<__half*>(dst + off) = h;
            *reinterpret_cast<__half*>(dst + HALF_STRIDE + off) = __float2half_rn(v * sw - __half2float(h));
        } else {
            *reinterpret_cast<__half*>(dst + off) = __float2half_rn(v);
        }
    }
}

size_t mlp_wg_packed_bytes(bool split) { return wg::image_bytes(split); }

int pack_mlp_wg(const float* const* w, bool split, void* packed, cudaStream_t stream) {
    MlpPtrsWg p;
    for (int i = 0; i < MVSN_N_MLP_TENSORS; ++i) p.p[i] = w[i];
    if (split) {
        uint8_t* wmax = static_cast<uint8_t*>(packed) + wg::tail_offset(true) + wg::BIAS_WMAX * 4;
        MVSN_CUDA_CHECK(cudaMemsetAsync(wmax, 0, 4, stream));
        wmax_mlp_wg_kernel<<<wg::NCHUNK, 256, 0, stream>>>(p, static_cast<uint8_t*>(packed));
        MVSN_CUDA_CHECK(cudaGetLastError());
    }
    pack_mlp_wg_kernel<<<wg::NCHUNK + 1, 256, 0, stream>>>(p, split, static_cast<uint8_t*>(packed));
    MVSN_CUDA_CHECK(cudaGetLastError());
    return MVSN_OK;
}

}  // namespace mvsn
