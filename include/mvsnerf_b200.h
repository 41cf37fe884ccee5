/*
 * mvsnerf_b200 -- C ABI of the H100-native (sm_90a) MVSNeRF render hot path.
 *
 * The reference (apchenstu/mvsnerf) has no FFI layer: the hot path sits behind
 * plain Python callables (SURVEY.md 8(b)).  Each entry point below replaces the
 * arithmetic of one of those callables; the Python mirror of the reference's
 * call signatures lives in mvsnerf_b200/backend.py and binds this header with
 * ctypes (INTEGRATION.md shows the stub a reference maintainer would add).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name ends in `_host`;
 *   - all tensors are dense fp32 unless stated, layouts are written as C arrays;
 *   - the caller owns every buffer (including workspaces); the library allocates
 *     nothing and keeps no state between calls;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it and
 *     the call returns without synchronising;
 *   - return value: 0 on success, a negative MVSN_E* code otherwise; the text of
 *     the last error on the calling thread is available from mvsn_last_error();
 *     nothing ever throws across this boundary.
 */
#ifndef MVSNERF_B200_H
#define MVSNERF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MVSN_OK          0
#define MVSN_EBADSHAPE  -1   /* illegal size (e.g. padded volume dims not divisible by 8)   */
#define MVSN_EALIGN     -2   /* pointer not 16-byte aligned where the kernel needs it       */
#define MVSN_ECUDA      -3   /* a CUDA call failed; see mvsn_last_error()                   */
#define MVSN_ENULL      -4   /* required pointer is NULL                                    */
#define MVSN_EWORKSPACE -5   /* workspace too small                                         */
#define MVSN_EUNSUPPORTED -6 /* feature/mode not available                                  */

/* arithmetic modes of the per-sample MLP (the GEMMs inside the render kernel) */
#define MVSN_MLP_FP32        0  /* fp32 FFMA, parity <= 1e-4 RGB Linf (north-star fp32 gate)        */
#define MVSN_MLP_TC_HALF     1  /* wgmma fp16 operands, fp32 accumulate, gate 5e-3                 */
#define MVSN_MLP_TC_SPLIT    2  /* wgmma, 2-term fp16 operand split (3 MMAs), fp32-grade, 1e-4      */
#define MVSN_MLP_TC_PAIR     3  /* same kernel and image as TC_HALF (the bench headline): weights     */
                                /* streamed, activations in registers, views/feature layers folded  */
                                /* (TC modes take any N_samples; rays are tiled up to 32 at a time)    */
/* grad_mode of the rays fine-tuning entries only (mvsn_render_backward_rays / _rays_stop and their workspace sizes):
 * MVSN_MLP_TC_HALF's backward plus the forward recompute's MLP on wgmma.  GEMMs with N >= 64 (pts_bias, layers 0-5,
 * feature_linear, the 128 feature columns of views_linears.0) take fp16 operands with fp32 accumulation; hidden
 * activations carry an exact power-of-two scale per sample row (row maximum in [2^14, 2^15)), the encoding and the 20
 * features are unscaled, weights are rounded unscaled, conversions saturate; layer 5's encoding and h parts are
 * combined by an exact power-of-two rescale.  alpha_linear, rgb_linear and the view-direction columns stay FFMA on
 * operands rounded to fp16's significand; biases, modulation, activations, compositing and the front end stay fp32.
 * A row's result depends on that row only: a ray's rgb, depth and loss term do not depend on the other rays of the
 * batch, and the early-termination recompute repeats the first bit for bit.  rgb is within the 5e-3 tier of
 * MVSN_MLP_FP32. */
#define MVSN_GRAD_TC_FULL    4
#define MVSN_VOLUME_F16      0x100 /* flag OR-ed into mvsn_render_scene.mlp_mode with a TC mode: volume_dhwc points at an */
                                /* fp16 [D,Hp,Wp,8] image (16-byte aligned).  Each value is widened exactly to fp32, so a  */
                                /* render is bit-identical to one from the fp32 volume vol.half().float(); the storage     */
                                /* rounding is the only change.  Render entries only: with MVSN_MLP_FP32 and in every      */
                                /* mvsn_render_backward* entry it gives MVSN_EUNSUPPORTED before any CUDA call;            */
                                /* mvsn_mlp_pack / mvsn_mlp_packed_bytes ignore it.                                         */

#define MVSN_N_MLP_TENSORS   22 /* network_fn_state_dict, reference models.py:145-222 / SURVEY App. B */
#define MVSN_N_COSTREG_TENSORS 30 /* 10 x (conv weight, bn gamma, bn beta), models.py:725-769          */
#define MVSN_N_FEATURENET_TENSORS 26 /* 8 x (conv weight, bn gamma, bn beta) + toplayer (weight, bias)   */
#define MVSN_VOL_CH          8
#define MVSN_MAX_PEERS       16 /* ranks of one NVLink domain a frame sink can address              */
#define MVSN_COST_CH         41
#define MVSN_FEAT_CH         32

const char* mvsn_last_error(void);
int mvsn_abi_version(void);

/* ---------------------------------------------------------------------------------------
 * MLP weights  (replaces: nn.Linear parameter reads in Renderer_ours.forward, models.py:194-222)
 *
 * w[22]: device pointers in this order (PyTorch [out,in] row-major, exactly the tensors of
 *   network_fn_state_dict):  pts_linears.{0..5}.weight/.bias interleaved (w0,b0,...,w5,b5),
 *   pts_bias.weight, pts_bias.bias, views_linears.0.weight, .bias, feature_linear.weight, .bias,
 *   alpha_linear.weight, .bias, rgb_linear.weight, .bias.
 * Re-call after every optimiser step when fine-tuning (cost: one small kernel).
 * ------------------------------------------------------------------------------------- */
size_t mvsn_mlp_packed_bytes(int mode);
int mvsn_mlp_pack(const float* const* w_host_array_of_device_ptrs, int mode,
                  void* packed, size_t packed_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Layout helpers
 *   images  [V,3,H,W] (planar, un-normalised [0,1])  ->  [V,H,W,4] (r,g,b,0) texel-interleaved
 *   volume  [8,D,Hp,Wp] (reference layout)           ->  [D,Hp,Wp,8] channels-last
 * The render kernel reads only the interleaved forms (one 16/32-byte sector per tap).
 * ------------------------------------------------------------------------------------- */
int mvsn_pack_images(const float* imgs, int V, int H, int W, float* imgs_hwc4, void* stream);
int mvsn_volume_to_channels_last(const float* vol_cdhw, int D, int Hp, int Wp,
                                 float* vol_dhwc, void* stream);
int mvsn_volume_from_channels_last(const float* vol_dhwc, int D, int Hp, int Wp,
                                   float* vol_cdhw, void* stream);
/* fp16 volume image for MVSN_VOLUME_F16: src is planar [8,D,Hp,Wp] (src_planar != 0) or channels-last [D,Hp,Wp,8],
 * fp32 or fp16 (src_half != 0), dense, aligned to its element size; vol_dhwc_f16 [D,Hp,Wp,8] fp16, 16-byte aligned.
 * fp32 values are rounded with __float2half_rn, as Tensor.half() rounds them: beyond 65504 they become inf and fp16
 * subnormals are kept.  Argument errors are returned before any CUDA call. */
int mvsn_volume_to_half(const void* src, int src_half, int src_planar, int D, int Hp, int Wp, void* vol_dhwc_f16,
                        void* stream);

/* ---------------------------------------------------------------------------------------
 * Rendering  (replaces: renderer.rendering, renderer.py:138-165, and everything it calls:
 *   gen_dir_feature :111-122, gen_pts_feats :124-136, utils.index_point_feature utils.py:357-383,
 *   utils.build_color_volume utils.py:300-332, run_network_mvs renderer.py:42-63,
 *   Embedder.embed models.py:47-51, Renderer_ours.forward models.py:194-222,
 *   raw2outputs/raw2alpha renderer.py:18-26,65-92)
 * ------------------------------------------------------------------------------------- */
typedef struct mvsn_render_scene {
    const float* volume_dhwc;   /* [D,Hp,Wp,8] channels-last encoding volume (fp16 with MVSN_VOLUME_F16) */
    int D, Hp, Wp;
    const float* imgs_hwc4;     /* [V,H,W,4] source images, from mvsn_pack_images               */
    int V, H, W;                /* V must be 3 (feat_dim = 8 + 4V = 20, train_mvs_nerf_pl.py:38) */
    const float* w2cs;          /* [V,4,4] device: world -> camera, pose_source['w2cs']           */
    const float* intrinsics;    /* [V,3,3] device: full-resolution K, pose_source['intrinsics']   */
    const void* mlp_packed;     /* from mvsn_mlp_pack                                             */
    int mlp_mode;               /* MVSN_MLP_*, optionally | MVSN_VOLUME_F16 (TC modes)            */
    int white_bkgd;             /* renderer.py:91-92                                              */
} mvsn_render_scene;

/* Signature-compatible entry: the caller has already run ray_marcher and get_ndc_coordinate.
 *   rays_pts [N,S,3] world points, rays_ndc [N,S,3] volume coords in [0,1], z_vals [N,S],
 *   rays_dir [N,3] (un-normalised).
 * Outputs: rgb [N,3], depth [N] required; weights [N,S], alpha [N,S], input_feat [N,S,20]
 * optional (NULL to skip).  */
int mvsn_render_samples(const mvsn_render_scene* scene,
                        const float* rays_pts, const float* rays_ndc, const float* z_vals,
                        const float* rays_dir, int N, int S,
                        float* rgb, float* depth, float* weights, float* alpha, float* input_feat,
                        void* stream);

/* mvsn_render_samples_stop: mvsn_render_samples (rgb and depth only) with early ray termination, by the rule of
 * mvsn_render_rays_stop: rays are composited in groups of up to 32 neighbours; after compositing tile k of a group, if
 * every ray of the group has transmittance T < t_stop, the group's tiles k + 3 onwards are not computed and each pixel
 * is the prefix of mvsn_render_samples' sums (same order, same arithmetic).  The omitted tail weighs less than t_stop:
 * per channel, -t_stop < rgb - rgb_full <= 0 (white_bkgd: 0 <= rgb - rgb_full < t_stop), 0 <= depth_full - depth <
 * t_stop * max z_vals.  t_stop = 0 never stops (bit-identical to mvsn_render_samples).  A group's result depends on its
 * own rays only.  tiles_done (device, 8-byte aligned, may be NULL): += the number of 64-sample tiles computed.  Inputs
 * as mvsn_render_samples; weights, alpha and input_feat are not computed (dead samples have none).
 * Modes MVSN_MLP_TC_HALF / TC_PAIR / TC_SPLIT (optionally | MVSN_VOLUME_F16); MVSN_MLP_FP32 gives MVSN_EUNSUPPORTED.
 * Argument errors (NULL pointers, t_stop negative or NaN, the mode, a misaligned tiles_done) are returned before any
 * CUDA call. */
int mvsn_render_samples_stop(const mvsn_render_scene* scene,
                             const float* rays_pts, const float* rays_ndc, const float* z_vals,
                             const float* rays_dir, int N, int S, float t_stop,
                             float* rgb, float* depth, unsigned long long* tiles_done, void* stream);

/* Fused-caller entry: also replaces data/ray_utils.ray_marcher (data/ray_utils.py:152-197,
 * perturb = 0) and utils.get_ndc_coordinate (utils.py:112-146) for the reference camera.
 *   rays [N,8] = (origin, direction, near, far); t_steps [S] = linspace(0,1,S) as the caller's
 *   framework computes it (kept as an input so z_vals match it bit for bit);
 *   ndc_near/ndc_far: the source views' near_far; pad: cost-volume padding in feature pixels
 *   (callers pass pad * imgScale_test); lindisp as in the reference. */
typedef struct mvsn_ray_params {
    float ndc_near, ndc_far;
    float pad;
    int lindisp;
} mvsn_ray_params;

int mvsn_render_rays(const mvsn_render_scene* scene, const mvsn_ray_params* rp,
                     const float* rays, const float* t_steps, int N, int S,
                     float* rgb, float* depth, float* weights, float* alpha, float* input_feat,
                     void* stream);

/* mvsn_render_rays_stop: mvsn_render_rays (rgb and depth only) with early ray termination.  Rays are composited in
 * groups of up to 32 neighbours, two samples per tile at frame sizes; after compositing tile k of a group, if every ray
 * of the group has transmittance T < t_stop, the group's tiles k + 3 onwards are not computed and each pixel is the
 * prefix of mvsn_render_rays' sums (same order, same arithmetic).  The omitted tail weighs less than t_stop: per
 * channel, -t_stop < rgb - rgb_full <= 0 (white_bkgd: 0 <= rgb - rgb_full < t_stop), 0 <= depth_full - depth <
 * t_stop * far.  t_stop = 0 never stops (bit-identical to mvsn_render_rays).  A group's result depends on its own rays
 * only, so frames are bit-reproducible.  tiles_done (device, 8-byte aligned, may be NULL): += the number of 64-sample
 * tiles computed.
 * Modes MVSN_MLP_TC_HALF / TC_PAIR / TC_SPLIT; MVSN_MLP_FP32 gives MVSN_EUNSUPPORTED.  Argument errors (NULL pointers,
 * t_stop negative or NaN, the mode, a misaligned rays or tiles_done) are returned before any CUDA call. */
int mvsn_render_rays_stop(const mvsn_render_scene* scene, const mvsn_ray_params* rp,
                          const float* rays, const float* t_steps, int N, int S, float t_stop,
                          float* rgb, float* depth, unsigned long long* tiles_done, void* stream);

/* Empty-space skipping.  An occupancy grid holds one bit per cell of the scene's D x Hp x Wp encoding-volume node grid
 * in NDC: bit c = (d * Hp + y) * Wp + x of the 32-bit word c / 32, least significant bit first,
 * mvsn_occupancy_bytes(D, Hp, Wp) = 4 * ceil(D * Hp * Wp / 32) bytes (586 KB at 512x640, pad 24).  Cell (d, y, x) with
 * d < D - 1, y < Hp - 1, x < Wp - 1 spans the nodes d..d+1, y..y+1, x..x+1; the other bits are 0.
 *
 * mvsn_build_occupancy evaluates the density at every node (NDC = the node; the world point inverts
 * utils.get_ndc_coordinate for rp, pad and lindisp included) with the samples entry in MVSN_MLP_TC_SPLIT, sets a cell
 * when alpha = 1 - exp(-sigma) > 0 at any of its eight corner nodes, then dilates by `dilate` cells (a (2 dilate + 1)^3
 * box).  scene->mlp_mode must be MVSN_MLP_TC_SPLIT (| MVSN_VOLUME_F16: fp32 and fp16 volumes); scene->white_bkgd is
 * unused; D, Hp, Wp >= 2; 0 <= dilate <= 8.  bits: mvsn_occupancy_bytes, 4-byte aligned, OVERWRITTEN.  Workspace:
 * mvsn_build_occupancy_workspace_bytes(D, Hp, Wp) bytes, 16-byte aligned (0 for D, Hp or Wp < 2).  The grid depends on
 * the volume, the MLP, the source images and cameras and rp: rebuild it after fine-tuning.  Argument errors are
 * returned before any CUDA call. */
typedef struct mvsn_occupancy {
    const uint32_t* bits;       /* device, 4-byte aligned */
    int D, Hp, Wp;              /* must equal the scene's volume dims */
} mvsn_occupancy;

size_t mvsn_occupancy_bytes(int D, int Hp, int Wp);
size_t mvsn_build_occupancy_workspace_bytes(int D, int Hp, int Wp);
int mvsn_build_occupancy(const mvsn_render_scene* scene, const mvsn_ray_params* rp, int dilate, uint32_t* bits,
                         void* workspace, size_t workspace_bytes, void* stream);

/* mvsn_render_rays_occ: mvsn_render_rays_stop with empty-space skipping.  A pre-pass marches every ray with the render
 * kernel's own ray march and NDC and gives each group of rays the range [k_first, k_last] of the tiles that hold a
 * sample in an occupied cell (a sample outside [0,1]^3 counts as occupied); the group computes only that range, with
 * the t_stop rule counted in computed tiles, and a group with no occupied sample stores rgb 0 (1 with white_bkgd) and
 * depth 0 without computing a tile.  Inside the range the arithmetic is mvsn_render_rays_stop's, so a pixel is
 * bit-identical to the full render whenever the full render's alpha is exactly 0 on every skipped sample; otherwise,
 * with A = 1 - prod over the skipped leading samples of (1 - alpha), each channel differs by at most A plus the
 * transmittance left after k_last, plus the t_stop bound.  The grid is a heuristic: these are properties of the scene,
 * not guarantees.  An all-ones grid with t_stop gives exactly mvsn_render_rays_stop's results.  tiles_done as there.
 * Modes MVSN_MLP_TC_HALF / TC_PAIR / TC_SPLIT.  Workspace (the range table): mvsn_render_rays_occ_workspace_bytes(N, S)
 * bytes, 16-byte aligned.  Argument errors are returned before any CUDA call: those of mvsn_render_rays_stop, a NULL or
 * misaligned grid, grid dims other than the scene's (MVSN_EBADSHAPE), a small or misaligned workspace. */
size_t mvsn_render_rays_occ_workspace_bytes(int N, int S);
int mvsn_render_rays_occ(const mvsn_render_scene* scene, const mvsn_ray_params* rp,
                         const float* rays, const float* t_steps, int N, int S, float t_stop,
                         const mvsn_occupancy* occupancy, float* rgb, float* depth, unsigned long long* tiles_done,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Importance sampling from a density grid (the reference's --use_density_volume --N_importance K).
 *
 * mvsn_build_density: sigma = relu(alpha_linear(h)) in fp32 at every node of the scene's D x Hp x Wp grid, laid out
 * [D][Hp][Wp] (the shape of the reference's density_volume).  The nodes are mvsn_build_occupancy's (NDC = the node, the
 * world point inverts utils.get_ndc_coordinate for rp), evaluated by the fp32 FFMA tile of MVSN_MLP_FP32.
 * scene->mlp_mode must be MVSN_MLP_FP32 (| MVSN_VOLUME_F16: an fp16 volume image, whose grid equals the one of its fp32
 * upcast bit for bit); scene->white_bkgd is unused; D, Hp, Wp >= 2.  sigma: D * Hp * Wp floats, 4-byte aligned,
 * OVERWRITTEN.  Workspace: mvsn_build_density_workspace_bytes(D, Hp, Wp) bytes, 16-byte aligned (0 for a dim < 2).
 * Argument errors are returned before any CUDA call.
 *
 * mvsn_sample_importance: data/ray_utils.ray_marcher_fine + sample_pdf for N rays [N,8] (16-byte aligned).  The S
 * coarse depths come from one of two sources:
 *   t_steps [S] (+ optional jitter [N,S]): marched from each ray's near / far as mvsn_render_backward_rays marches them,
 *     their NDC by the render's get_ndc_coordinate (scene's reference camera, rp);  z_vals and ndc NULL;
 *   z_vals [N,S] (nondecreasing or not) and ndc [N,S,3]: the caller's;  t_steps and jitter NULL.
 * sigma_j is the grid's trilinear value at the sample's NDC (align_corners, zero padding; the NDC itself, not the
 * reference's doubled 4 ndc - 3 mapping), alpha_j = 1 - exp(-relu(sigma_j)), w_j = alpha_j prod_{i<j}(1 - alpha_i + 1e-10),
 * and K depths are drawn by inverse-CDF sampling of (w_1..w_{S-2} + 1e-5) over the midpoints of the coarse depths with
 * u [N,K] (NULL: torch.linspace(0, 1, K) for every ray).  Outputs: z_out [N,S+K] = sort(cat(fine, coarse)) ascending
 * (NaN last; the coarse values bit-exact), pts_out [N,S+K,3] = o + d * z (multiply, then add), ndc_out [N,S+K,3]
 * (optional) their NDC.  scene and rp are needed by the march and ndc_out only (may be NULL otherwise); with a scene,
 * the grid's dims must equal its volume's.  3 <= S, 1 <= K (MVSN_EBADSHAPE), S + K <= 1024 (MVSN_EUNSUPPORTED).
 * Argument errors are returned before any CUDA call. */
typedef struct mvsn_density {
    const float* sigma;         /* device [D][Hp][Wp] fp32, 4-byte aligned */
    int D, Hp, Wp;
} mvsn_density;

size_t mvsn_build_density_workspace_bytes(int D, int Hp, int Wp);
int mvsn_build_density(const mvsn_render_scene* scene, const mvsn_ray_params* rp, float* sigma, void* workspace,
                       size_t workspace_bytes, void* stream);
int mvsn_sample_importance(const mvsn_render_scene* scene, const mvsn_ray_params* rp, const mvsn_density* density,
                           const float* rays, const float* t_steps, const float* jitter, const float* z_vals,
                           const float* ndc, const float* u, int N, int S, int K, float* z_out, float* pts_out,
                           float* ndc_out, void* stream);

/* Ray generation for one camera (replaces: data/ray_utils.get_rays, data/ray_utils.py:32-53, and the notebooks'
 * `torch.cat([rays_o, rays_d, near, far])`): directions [n,3] = get_ray_directions(H, W, focal) in camera coordinates
 * (resident on the device, they depend on the intrinsics only), c2w = the first three rows of the camera-to-world matrix,
 * row-major with row stride 4 ([3,4] or [4,4]), on the device.  rays [n,8] = (c2w[:3,3], directions @ c2w[:3,:3]^T,
 * near, far): the input of mvsn_render_rays, so a frame needs 48 bytes of host input. */
int mvsn_make_rays(const float* directions, const float* c2w, float near, float far, int n, float* rays, void* stream);

/* ---------------------------------------------------------------------------------------
 * Fine-tuning step  (replaces: autograd through renderer.rendering + torch.optim.Adam in
 *   train_mvs_nerf_finetuning_pl.py:140-189 -- gradients of the 22 MLP tensors, models.py:145-222, and of
 *   RefVolume.feat_volume, models.py:935-950 -- SURVEY.md 8(f) row 2).
 *
 * mvsn_render_backward re-evaluates the samples in fp32 and back-propagates the given output gradients in one
 * kernel: reverse compositing scan, MLP dgrad/wgrad, trilinear scatter-add into the volume gradient.
 *   scene->mlp_packed must be the MVSN_MLP_FP32 image (scene->mlp_mode == MVSN_MLP_FP32);
 *   mlp_w[22]: the live nn.Linear tensors (device pointers, order as mvsn_mlp_pack);
 *   inputs as mvsn_render_samples; N_samples <= 128;
 *   g: output gradients.  Either g->rgb [N,3] (d loss / d rgb_map) or g->target_rgb [N,3] with g->loss_scale =
 *      1 / (3 * N_total): the img2mse loss and its gradient are then formed in the kernel (g->loss_out, if set, is
 *      ACCUMULATED with this call's share of the loss; g->rgb_out / g->depth_out receive the forward result).
 *      g->depth [N], g->weights [N,S], g->alpha [N,S], g->input_feat [N,S,20] optional (NULL = zero).
 *   grad_mlp[22]: OVERWRITTEN with d loss / d tensor, nn.Linear layouts;
 *   grad_volume_dhwc: [D,Hp,Wp,8] channels-last, ACCUMULATED (atomics); NULL = volume frozen;
 *   workspace: mvsn_render_backward_workspace_bytes(N, S) bytes, 16-byte aligned.
 * Every mvsn_render_backward* entry returns its argument errors before any CUDA call, checked in this order: a
 *   grad_mode the entry does not take (MVSN_EUNSUPPORTED); the scene; NULL pointers (MVSN_ENULL); with t_stop (the
 *   _stop entries), t_stop negative, NaN or > 1 (MVSN_EBADSHAPE), then g->weights / g->alpha / g->input_feat set
 *   (MVSN_EUNSUPPORTED: per-sample cotangents of dead samples are not defined); a misaligned rays, grad_volume_dhwc,
 *   live_samples or tiles_done (MVSN_EALIGN); N < 0 or N_samples < 1 (MVSN_EBADSHAPE); N_samples > 128
 *   (MVSN_EUNSUPPORTED); scene->mlp_packed not the MVSN_MLP_FP32 image (MVSN_EUNSUPPORTED).  N == 0 then returns
 *   MVSN_OK.
 * mvsn_adam_step / mvsn_adam_step_volume: torch.optim.Adam arithmetic (betas, eps, bias correction by `step` >= 1,
 *   no weight decay / amsgrad).  The volume variant reads the channels-last gradient, zeroes it for the next step,
 *   and updates a parameter (and moments) stored channels-last (planar = 0) or planar [8][nvox] (planar = 1).
 * ------------------------------------------------------------------------------------- */
typedef struct mvsn_render_grads {
    const float* rgb;
    const float* target_rgb;
    float loss_scale;
    const float* depth;
    const float* weights;
    const float* alpha;
    const float* input_feat;
    float* rgb_out;
    float* depth_out;
    float* loss_out;
} mvsn_render_grads;

size_t mvsn_render_backward_workspace_bytes(int N, int S);
int mvsn_render_backward(const mvsn_render_scene* scene, const float* const* mlp_w,
                         const float* rays_pts, const float* rays_ndc, const float* z_vals, const float* rays_dir,
                         int N, int S, const mvsn_render_grads* g, float* const* grad_mlp, float* grad_volume_dhwc,
                         void* workspace, size_t workspace_bytes, void* stream);
/* mvsn_render_backward_tc: the same call, arguments and outputs as mvsn_render_backward (scene->mlp_packed is still
 * the MVSN_MLP_FP32 image, used by the forward recompute; N_samples <= 128, otherwise MVSN_EUNSUPPORTED), with the
 * MLP dgrad / wgrad GEMMs on tensor cores: dpre, layer inputs and weights rounded to fp16 (each tile with an exact
 * power-of-two scale), fp32 accumulation.  rgb_out / depth_out are bit-identical to mvsn_render_backward's, and so is
 * each ray's loss term (loss_out sums them with float atomics); gradients agree with it to ~1e-3 of their max |g|.  Workspace: mvsn_render_backward_tc_workspace_bytes(N, S). */
size_t mvsn_render_backward_tc_workspace_bytes(int N, int S);
int mvsn_render_backward_tc(const mvsn_render_scene* scene, const float* const* mlp_w,
                            const float* rays_pts, const float* rays_ndc, const float* z_vals, const float* rays_dir,
                            int N, int S, const mvsn_render_grads* g, float* const* grad_mlp, float* grad_volume_dhwc,
                            void* workspace, size_t workspace_bytes, void* stream);
/* mvsn_render_backward_deterministic: mvsn_render_backward (grad_mode MVSN_MLP_FP32) or mvsn_render_backward_tc
 * (MVSN_MLP_TC_HALF) with every output bit-reproducible from call to call on the same GPU model and inputs.  The
 * backward kernel records each sample's 8 volume-feature gradients and each ray's loss term instead of adding them
 * with float atomics; the volume gradient is then summed as 64-bit fixed-point integers at a power-of-two scale chosen
 * from the largest |gradient| (contributions below ~max|g| * N * S * 2^-62 round to zero) and ACCUMULATED into
 * grad_volume_dhwc, and loss_out is ACCUMULATED with the per-ray terms summed in a fixed order.  rgb_out / depth_out
 * and the MLP gradients are the same as the non-deterministic entry's.  A non-finite gradient makes the volume
 * entries it touches NaN / inf as the atomics would.  Any other grad_mode (MVSN_GRAD_TC_FULL included: rays entries
 * only): MVSN_EUNSUPPORTED, before any CUDA call.
 * Workspace: mvsn_render_backward_deterministic_workspace_bytes(N, S, D, Hp, Wp, grad_mode), 16-byte aligned, with the
 * scene's volume dims (it holds a [D,Hp,Wp,8] int64 accumulator, zeroed by every call); D = Hp = Wp = 0 sizes it for a
 * frozen volume (grad_volume_dhwc = NULL).  0 for an unknown grad_mode or shape. */
size_t mvsn_render_backward_deterministic_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode);
int mvsn_render_backward_deterministic(const mvsn_render_scene* scene, const float* const* mlp_w,
                                       const float* rays_pts, const float* rays_ndc, const float* z_vals,
                                       const float* rays_dir, int N, int S, int grad_mode, const mvsn_render_grads* g,
                                       float* const* grad_mlp, float* grad_volume_dhwc, void* workspace,
                                       size_t workspace_bytes, void* stream);
/* mvsn_render_backward_rays: the fine-tuning step straight from rays, as train_mvs_nerf_finetuning_pl.py:140-164 feeds
 * it -- the backward kernel also replaces data/ray_utils.ray_marcher (with perturb) and utils.get_ndc_coordinate, so
 * no per-sample array is read.  rays [N,8], t_steps [S] and rp as mvsn_render_rays (rays 16-byte aligned);
 * jitter [N,S] = perturb * u, u uniform in [0,1) as the caller's RNG draws it (NULL: no jitter, the depths are exactly
 * mvsn_render_rays'): sample s of a ray lies at lower + (upper - lower) * jitter, between the midpoints of the
 * neighbouring unjittered depths (data/ray_utils.py:184-191), each operation rounded as fp32 element-wise ops round it.
 * grad_mode MVSN_MLP_FP32 or MVSN_MLP_TC_HALF selects the arithmetic of the GEMMs as mvsn_render_backward /
 * mvsn_render_backward_tc do, MVSN_GRAD_TC_FULL also moves the forward recompute to tensor cores (see its define;
 * rgb_out / depth_out / the loss are then this mode's forward); deterministic != 0 sums the volume gradient and the loss as
 * mvsn_render_backward_deterministic does.  g, grad_mlp and grad_volume_dhwc as mvsn_render_backward; rgb_out /
 * depth_out receive the forward of the marched samples (with jitter = NULL: rgb bit-identical to mvsn_render_rays with
 * the MVSN_MLP_FP32 image).  N_samples <= 128.  Argument errors: see the head of this section.
 * Workspace: mvsn_render_backward_rays_workspace_bytes(N, S, D, Hp, Wp, grad_mode, deterministic) bytes, 16-byte
 * aligned; the volume dims matter only with `deterministic` (D = Hp = Wp = 0: a frozen volume).  0 for an unknown
 * grad_mode or shape. */
size_t mvsn_render_backward_rays_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode, int deterministic);
int mvsn_render_backward_rays(const mvsn_render_scene* scene, const float* const* mlp_w, const mvsn_ray_params* rp,
                              const float* rays, const float* t_steps, const float* jitter, int N, int S, int grad_mode,
                              int deterministic, const mvsn_render_grads* g, float* const* grad_mlp,
                              float* grad_volume_dhwc, void* workspace, size_t workspace_bytes, void* stream);
/* mvsn_render_backward_rays_stop: mvsn_render_backward_rays with early ray termination.  For each ray, with alpha_j
 * from this mode's recompute, T_0 = 1 and T_{j+1} = T_j ((1 - alpha_j) + 1e-10) (the kernel's fp32 order), sample j is
 * live iff T_j >= t_stop; the live samples are a prefix of length L (L >= 1).  The step renders, forms the loss of and
 * exactly differentiates the truncated render sum_{j<L} w_j c_j (depth and white_bkgd likewise); dead samples get no
 * gradient and no volume scatter.  Against the full render, per channel -t_stop < rgb - rgb_full <= 0 (white_bkgd:
 * 0 <= rgb - rgb_full < t_stop) and 0 <= depth_full - depth < t_stop * far, up to a few ulps.  t_stop = 0 keeps every
 * sample: every output is bit-identical to mvsn_render_backward_rays.  With MVSN_MLP_FP32 or MVSN_GRAD_TC_FULL a ray's rgb, depth
 * and loss term do not depend on the other rays of the batch; the MLP gradients may differ from a differently packed batch in
 * summation order only.  deterministic != 0: every output is a deterministic function of the inputs.
 * live_samples [N] int32 (device, 4-byte aligned, may be NULL): each ray's L.  tiles_done (device, 8-byte aligned, may
 * be NULL): unsigned long long[3] += the 128-row tiles back-propagated immediately, deferred, and packed from deferred
 * rays.  Everything else as mvsn_render_backward_rays; argument errors: see the head of this section.  Workspace:
 * mvsn_render_backward_rays_stop_workspace_bytes(N, S, D, Hp, Wp, grad_mode, deterministic) bytes, 16-byte aligned (a
 * little more than mvsn_render_backward_rays'). */
size_t mvsn_render_backward_rays_stop_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode,
                                                      int deterministic);
int mvsn_render_backward_rays_stop(const mvsn_render_scene* scene, const float* const* mlp_w, const mvsn_ray_params* rp,
                                   const float* rays, const float* t_steps, const float* jitter, int N, int S,
                                   int grad_mode, int deterministic, float t_stop, const mvsn_render_grads* g,
                                   float* const* grad_mlp, float* grad_volume_dhwc, int* live_samples,
                                   unsigned long long* tiles_done, void* workspace, size_t workspace_bytes, void* stream);
/* mvsn_render_backward_stop: mvsn_render_backward (grad_mode MVSN_MLP_FP32) or mvsn_render_backward_tc
 * (MVSN_MLP_TC_HALF) with early ray termination, by the rule of mvsn_render_backward_rays_stop: for each ray, with
 * alpha_j from the fp32 recompute, T_0 = 1 and T_{j+1} = T_j ((1 - alpha_j) + 1e-10) (the kernel's fp32 order), sample
 * j is live iff T_j >= t_stop; the live samples are a prefix of length L (L >= 1).  The step renders, forms the loss of
 * and exactly differentiates the truncated render sum_{j<L} w_j c_j (depth and white_bkgd likewise); dead samples get
 * no gradient and no volume scatter.  Against the full render, per channel -t_stop < rgb - rgb_full <= 0 (white_bkgd:
 * 0 <= rgb - rgb_full < t_stop) and 0 <= depth_full - depth < t_stop * max z_vals, up to a few ulps.  t_stop = 0 keeps
 * every sample: every output is bit-identical to the entry without it (mvsn_render_backward / _tc, or
 * mvsn_render_backward_deterministic with deterministic != 0).  With MVSN_MLP_FP32 a ray's rgb, depth and loss term do
 * not depend on the other rays of the batch; the MLP gradients may differ from a differently packed batch in summation
 * order only.  deterministic != 0: every output is a deterministic function of the inputs, summed as
 * mvsn_render_backward_deterministic sums them.  Inputs, g, grad_mlp and grad_volume_dhwc as mvsn_render_backward;
 * N_samples <= 128.  live_samples [N] int32 (device, 4-byte aligned, may be NULL): each ray's L.  tiles_done (device,
 * 8-byte aligned, may be NULL): unsigned long long[3] += the 128-row tiles back-propagated immediately, deferred, and
 * packed from deferred rays.  grad_mode MVSN_MLP_FP32 or MVSN_MLP_TC_HALF; argument errors: see the head of this
 * section.  Workspace:
 * mvsn_render_backward_stop_workspace_bytes(N, S, D, Hp, Wp, grad_mode, deterministic) bytes, 16-byte aligned; the
 * volume dims matter only with `deterministic` (D = Hp = Wp = 0: a frozen volume).  0 for an unknown grad_mode or
 * shape. */
size_t mvsn_render_backward_stop_workspace_bytes(int N, int S, int D, int Hp, int Wp, int grad_mode, int deterministic);
int mvsn_render_backward_stop(const mvsn_render_scene* scene, const float* const* mlp_w, const float* rays_pts,
                              const float* rays_ndc, const float* z_vals, const float* rays_dir, int N, int S,
                              int grad_mode, int deterministic, float t_stop, const mvsn_render_grads* g,
                              float* const* grad_mlp, float* grad_volume_dhwc, int* live_samples,
                              unsigned long long* tiles_done, void* workspace, size_t workspace_bytes, void* stream);
int mvsn_adam_step(float* const* params, const float* const* grads, float* const* exp_avg, float* const* exp_avg_sq,
                   const int* numel_host, int count, float lr, float beta1, float beta2, float eps, int step,
                   void* stream);
int mvsn_adam_step_volume(float* param, float* grad_dhwc, float* exp_avg, float* exp_avg_sq, long long nvox,
                          int planar, float lr, float beta1, float beta2, float eps, int step, void* stream);

/* ---------------------------------------------------------------------------------------
 * Multi-GPU frame assembly (replaces: nothing in the reference -- its DDP flag is dead code, SURVEY.md 2.3;
 * this is the north star's "rays shard across the GPUs of one box, the rendered image is gathered at the end",
 * SURVEY.md 8(e), done from the render kernel's epilogue instead of by a gather pass).
 *
 * A frame is [n_pixels][4] fp32 texels (r, g, b, depth).  Every rank owns one copy, allocated with
 * mvsn_peer_buffer_create (the ONE place this library allocates: the memory must be exportable to the other
 * processes), exports its 64-byte handle, and maps the other ranks' copies with mvsn_peer_buffer_open.
 * mvsn_render_rays_to_peers then renders this rank's band of rays and stores each finished pixel into all
 * `n_peers` copies (NVLink peer stores, 16 bytes per pixel per peer).  The frame is complete on every rank once
 * every rank's launch has completed (the caller orders that with any stream-level barrier).
 * rgb / depth may be NULL here (the sink is then the only output).
 * ------------------------------------------------------------------------------------- */
#define MVSN_PEER_HANDLE_BYTES 64
int mvsn_peer_buffer_create(size_t bytes, void** dev_ptr, unsigned char handle_host[MVSN_PEER_HANDLE_BYTES]);
int mvsn_peer_buffer_open(const unsigned char handle_host[MVSN_PEER_HANDLE_BYTES], void** peer_ptr);
int mvsn_peer_buffer_close(void* peer_ptr);
int mvsn_peer_buffer_destroy(void* dev_ptr);

typedef struct mvsn_peer_sink {
    float* frame[MVSN_MAX_PEERS]; /* frame[r]: rank r's copy, [n_pixels,4] fp32, 16-byte aligned (own or peer-mapped) */
    int n_peers;
    long long first_pixel;        /* index in the frame of this call's ray 0                                       */
} mvsn_peer_sink;

int mvsn_render_rays_to_peers(const mvsn_render_scene* scene, const mvsn_ray_params* rp,
                              const float* rays, const float* t_steps, int N, int S,
                              const mvsn_peer_sink* sink, float* rgb, float* depth, void* stream);

/* ---------------------------------------------------------------------------------------
 * Cost volume  (replaces: MVSNet.build_volume_costvar_img, models.py:839-893, with
 *   utils.homo_warp utils.py:580-630 and the F.interpolate at models.py:859)
 *   imgs   [V,3,H,W]  ImageNet-normalised source images (H = 4h, W = 4w)
 *   feats  [V,32,h,w] FeatureNet output
 *   proj   [V,3,4]    src_proj @ inv(ref_proj) in feature space (row 0 unused)
 *   depths [D]
 * Outputs (reference layouts): cost [41,D,h+2pad,w+2pad]; in_masks [V,D,h+2pad,w+2pad] or NULL.
 * The never-written pad border of channels 0:3 is defined as zero (SURVEY.md F5).
 * workspace: mvsn_cost_volume_workspace_bytes(V,h,w) bytes.
 * ------------------------------------------------------------------------------------- */
size_t mvsn_cost_volume_workspace_bytes(int V, int h, int w);
int mvsn_build_cost_volume(const float* imgs, const float* feats, const float* proj,
                           const float* depths, int V, int H, int W, int D, int pad,
                           float* cost, float* in_masks, void* workspace, size_t workspace_bytes,
                           void* stream);

/* ---------------------------------------------------------------------------------------
 * Feature extraction  (replaces: FeatureNet.forward + ConvBnReLU + InPlaceABN in train mode,
 *   models.py:661-672,688-722; called from MVSNet.forward models.py:907-909).
 *   w[26]: device pointers, for each of conv0.0, conv0.1, conv1.0, conv1.1, conv1.2, conv2.0, conv2.1,
 *          conv2.2 in that order: (conv weight [Cout,Cin,k,k], bn gamma, bn beta); then toplayer.weight
 *          [32,32,1,1] and toplayer.bias [32].
 *   imgs [V,3,H,W] (ImageNet-normalised) -> feats [V,32,ceil(H/4),ceil(W/4)].  Batch statistics are taken
 *   over all V views jointly, as the reference batches them (B*V images through one BN).
 * ------------------------------------------------------------------------------------- */
size_t mvsn_featurenet_workspace_bytes(int V, int H, int W);
int mvsn_featurenet_forward(const float* const* w_host_array_of_device_ptrs, const float* imgs,
                            int V, int H, int W, float* feats,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Cost regularisation  (replaces: CostRegNet.forward + ConvBnReLU3D + InPlaceABN in train mode,
 *   models.py:674-685,725-769).
 *   w[30]: device pointers, for each of conv0..conv6, conv7, conv9, conv11 in that order:
 *          (conv weight, bn gamma, bn beta).  conv weight layouts as in the checkpoint:
 *          Conv3d [Cout,Cin,3,3,3]; ConvTranspose3d [Cin,Cout,3,3,3].
 *   cost [41,D,Hp,Wp] -> volume_dhwc [D,Hp,Wp,8] (channels-last; use
 *   mvsn_volume_from_channels_last for the reference layout).  D, Hp, Wp must be divisible by 8.
 *   Batch statistics (every shipped caller runs MVSNet.train(), SURVEY.md F2); see mvsn_costreg_forward_bn for eval mode.
 * ------------------------------------------------------------------------------------- */
size_t mvsn_costreg_workspace_bytes(int D, int Hp, int Wp);
int mvsn_costreg_forward(const float* const* w_host_array_of_device_ptrs, const float* cost,
                         int D, int Hp, int Wp, float* volume_dhwc,
                         void* workspace, size_t workspace_bytes, void* stream);

/* BatchNorm mode of the two encoder entry points (InPlaceABN, models.py:661-685; `self.training` dispatch,
 * SURVEY.md 8(b)):
 *   MVSN_BN_BATCH         batch statistics, running statistics untouched (the plain entry points above);
 *   MVSN_BN_BATCH_UPDATE  batch statistics AND the train-mode side effect of F.batch_norm: running_mean / running_var
 *                         are updated in place with `momentum` (variance unbiased) -- what MVSNet.train()(...) does
 *                         to the buffers save_ckpt later serialises;
 *   MVSN_BN_RUNNING       eval mode: normalise with running_mean / running_var.
 * running[2 L]: for each BN layer in the order of w: (running_mean, running_var); L = 8 (FeatureNet), 10 (CostRegNet). */
#define MVSN_BN_BATCH         0
#define MVSN_BN_BATCH_UPDATE  1
#define MVSN_BN_RUNNING       2
#define MVSN_CONV0_FFMA       0x100 /* diagnostic flag, OR-ed into bn_mode of mvsn_costreg_forward_bn: run the first layer
                                       (41 -> 8 channels) on the fp32 FFMA kernel instead of the wgmma kernel */
int mvsn_featurenet_forward_bn(const float* const* w_host_array_of_device_ptrs, float* const* running, int bn_mode,
                               float momentum, const float* imgs, int V, int H, int W, float* feats,
                               void* workspace, size_t workspace_bytes, void* stream);
int mvsn_costreg_forward_bn(const float* const* w_host_array_of_device_ptrs, float* const* running, int bn_mode,
                            float momentum, const float* cost, int D, int Hp, int Wp, float* volume_dhwc,
                            void* workspace, size_t workspace_bytes, void* stream);
/* mvsn_costreg_forward_f16: mvsn_costreg_forward_bn with the volume written as fp16 [D,Hp,Wp,8] (16-byte aligned), each
 * value the fp32 result rounded with __float2half_rn (bit-identical to .half() of mvsn_costreg_forward_bn's volume; the
 * running statistics are updated identically): the input of MVSN_VOLUME_F16 renders without a conversion pass. */
int mvsn_costreg_forward_f16(const float* const* w_host_array_of_device_ptrs, float* const* running, int bn_mode,
                             float momentum, const float* cost, int D, int Hp, int Wp, void* volume_dhwc_f16,
                             void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------
 * Diagnostic: one 128 x N x K fp16 GEMM (fp32 accumulate) through the same wgmma building blocks
 * the fused render kernel uses.  A [128,K], B [N,K] fp16 row-major; Bc [N,16] optional extra K-step
 * (D += A[:,16:32] * Bc^T, the "bias" step); D [128,N] fp32.  Used by tests only.
 * ------------------------------------------------------------------------------------- */
int mvsn_selftest_umma(const void* A, const void* B, const void* Bc, int N, int K, float* D, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MVSNERF_B200_H */
