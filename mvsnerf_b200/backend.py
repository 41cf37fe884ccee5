"""Host-side mirror of the reference's Python surface for the render hot path.

Same names, argument meaning and return tuples as apchenstu/mvsnerf (SURVEY.md 8(b)):

    create_nerf_mvs(args, ...)                      models.py:569-654
    MVSNet(imgs, proj_mats, near_far, pad, ...)     models.py:771-932
    MVSNeRF / network_fn                            models.py:540-567 (Renderer_ours, :145-222)
    RefVolume                                       models.py:935-950
    rendering(args, pose_ref, rays_pts, ...)        renderer.py:138-165

so the reference's per-scene fine-tuning script (train_mvs_nerf_finetuning_pl.py) and the render notebooks run with
`from mvsnerf_b200.backend import create_nerf_mvs, rendering, RefVolume`.  What does NOT carry over: end-to-end
training of the encoder (train_mvs_nerf_pl.py back-propagates through MVSNet): the encoding-volume kernels are
forward-only, `MVSNet.forward` returns a volume without a graph and says so with a warning when called under
autograd, and `create_nerf_mvs` therefore leaves the encoder's parameters out of `grad_vars`.  The modules keep the
reference's parameter names, so `ckpts/mvsnerf-v0.tar` (and fine-tuned checkpoints) load with
`load_state_dict(strict=True)`.  All arithmetic of the path runs in libmvsnerf_b200.so (hand
written sm_90a CUDA, bound through ctypes); PyTorch here only owns device memory, streams and
parameters.  There is no CPU path: CPU tensors are rejected with a RuntimeError.

`render_rays` is the fused-caller entry (ray marching + NDC conversion also in the kernel) that
replaces the notebooks' per-chunk loop of ray_marcher -> get_ndc_coordinate -> rendering.
"""
from __future__ import annotations

import ctypes as C
import warnings
import weakref

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import lib as _lib

N_DEPTH_PLANES = 128     # models.py:914


# --------------------------------------------------------------------------------------------
# parameter containers with the reference's state_dict keys
# --------------------------------------------------------------------------------------------
class InPlaceABN(nn.Module):
    """BatchNorm + leaky-ReLU(0.01) with the affine weight used as |gamma|+eps (inplace_abn).

    A parameter container inside FeatureNet / CostRegNet (the CUDA kernels apply it while loading the next
    layer's input); forward() is the plain PyTorch statement of the op for stand-alone use."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, slope=0.01):
        super().__init__()
        self.eps, self.momentum, self.slope = eps, momentum, slope
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))
        self.register_buffer("running_mean", torch.zeros(num_features))
        self.register_buffer("running_var", torch.ones(num_features))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))

    def forward(self, x):
        y = F.batch_norm(x, self.running_mean, self.running_var, self.weight.abs() + self.eps, self.bias,
                         self.training, self.momentum, self.eps)
        return F.leaky_relu(y, self.slope)


class ConvBnReLU(nn.Module):
    def __init__(self, cin, cout, k=3, stride=1, pad=1):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=pad, bias=False)
        self.bn = InPlaceABN(cout)

    def forward(self, x):
        return self.bn(self.conv(x))


class ConvBnReLU3D(nn.Module):
    """Parameter container (conv.weight, bn.*); evaluated by mvsn_costreg_forward."""

    def __init__(self, cin, cout, stride=1):
        super().__init__()
        self.conv = nn.Conv3d(cin, cout, 3, stride=stride, padding=1, bias=False)
        self.bn = InPlaceABN(cout)


class FeatureNet(nn.Module):
    """models.py:688-722 parameter layout; forward = one C-ABI call (mvsn_featurenet_forward):
    eight conv + train-mode InPlaceABN layers (statistics over all views jointly) and the 1x1 toplayer."""

    def __init__(self):
        super().__init__()
        self.conv0 = nn.Sequential(ConvBnReLU(3, 8), ConvBnReLU(8, 8))
        self.conv1 = nn.Sequential(ConvBnReLU(8, 16, 5, 2, 2), ConvBnReLU(16, 16), ConvBnReLU(16, 16))
        self.conv2 = nn.Sequential(ConvBnReLU(16, 32, 5, 2, 2), ConvBnReLU(32, 32), ConvBnReLU(32, 32))
        self.toplayer = nn.Conv2d(32, 32, 1)

    def weight_list(self):
        out = []
        for block in (self.conv0, self.conv1, self.conv2):
            for m in block:
                out += [m.conv.weight, m.bn.weight, m.bn.bias]
        return out + [self.toplayer.weight, self.toplayer.bias]

    def bn_modules(self):
        return [m.bn for block in (self.conv0, self.conv1, self.conv2) for m in block]

    def forward(self, x):
        """x [V,3,H,W] -> [V,32,ceil(H/4),ceil(W/4)].  BatchNorm dispatches on `self.training` like InPlaceABN
        (models.py:661-672): train = batch statistics over the V views (+ running-statistics update), eval = running."""
        lib = _lib.load()
        x = _lib.dev_f32(x.detach(), "FeatureNet input")
        V, C, H, W = x.shape
        if C != 3:
            raise RuntimeError(f"FeatureNet expects [V,3,H,W] images, got {tuple(x.shape)}")
        ws_bytes = lib.mvsn_featurenet_workspace_bytes(V, H, W)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        feats = torch.empty(V, 32, (H + 3) // 4, (W + 3) // 4, dtype=torch.float32, device=x.device)
        weights = [_lib.dev_f32(w.detach(), "FeatureNet weight") for w in self.weight_list()]
        running, mode, momentum = _bn_call_args(self.bn_modules(), self.training)
        with torch.cuda.device(x.device):
            _lib.check(lib.mvsn_featurenet_forward_bn(_lib.ptr_array(weights), _lib.ptr_array(running), mode, momentum,
                                                      _lib.ptr(x), V, H, W, _lib.ptr(feats), _lib.ptr(ws), ws_bytes,
                                                      _lib.stream_ptr()), "mvsn_featurenet_forward_bn")
        return feats


def _bn_call_args(bns, training):
    """(running-statistics pointers, MVSN_BN_* mode, momentum) for a stack of InPlaceABN parameter containers."""
    running = []
    for bn in bns:
        for t in (bn.running_mean, bn.running_var):
            if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError("BatchNorm running statistics must be contiguous CUDA fp32 buffers")
            running.append(t)
    if not training:
        return running, _lib.BN_RUNNING, 0.0
    for bn in bns:
        bn.num_batches_tracked += 1                     # as nn.BatchNorm / InPlaceABN do in train mode
    return running, _lib.BN_BATCH_UPDATE, float(bns[0].momentum)


class CostRegNet(nn.Module):
    """models.py:725-769 parameter layout; forward = one C-ABI call."""

    LAYERS = ("conv0", "conv1", "conv2", "conv3", "conv4", "conv5", "conv6", "conv7", "conv9", "conv11")

    def __init__(self, in_channels=41):
        super().__init__()
        self.conv0 = ConvBnReLU3D(in_channels, 8)
        self.conv1 = ConvBnReLU3D(8, 16, stride=2)
        self.conv2 = ConvBnReLU3D(16, 16)
        self.conv3 = ConvBnReLU3D(16, 32, stride=2)
        self.conv4 = ConvBnReLU3D(32, 32)
        self.conv5 = ConvBnReLU3D(32, 64, stride=2)
        self.conv6 = ConvBnReLU3D(64, 64)
        for name, cin, cout in (("conv7", 64, 32), ("conv9", 32, 16), ("conv11", 16, 8)):
            setattr(self, name, nn.Sequential(
                nn.ConvTranspose3d(cin, cout, 3, padding=1, output_padding=1, stride=2, bias=False),
                InPlaceABN(cout)))

    def weight_list(self):
        out = []
        for name in self.LAYERS:
            m = getattr(self, name)
            conv, bn = (m.conv, m.bn) if isinstance(m, ConvBnReLU3D) else (m[0], m[1])
            out += [conv.weight, bn.weight, bn.bias]
        return out

    def bn_modules(self):
        out = []
        for name in self.LAYERS:
            m = getattr(self, name)
            out.append(m.bn if isinstance(m, ConvBnReLU3D) else m[1])
        return out

    def forward(self, cost, volume_dtype=torch.float32):
        """cost [1,41,D,Hp,Wp] (reference layout) -> [1,8,D,Hp,Wp] (channels-last memory).  BatchNorm dispatches on
        `self.training` (models.py:674-685): batch statistics (+ running update) in train mode, running in eval.
        volume_dtype=torch.float16: the volume is stored as fp16, bit-identical to .half() of the fp32 volume."""
        if volume_dtype not in (torch.float32, torch.float16):
            raise RuntimeError(f"CostRegNet: volume_dtype {volume_dtype} (torch.float32 or torch.float16)")
        lib = _lib.load()
        cost = _lib.dev_f32(cost, "cost volume")
        _, _, D, Hp, Wp = cost.shape
        ws_bytes = lib.mvsn_costreg_workspace_bytes(D, Hp, Wp)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=cost.device)
        vol = torch.empty(D, Hp, Wp, 8, dtype=volume_dtype, device=cost.device)
        weights = [_lib.dev_f32(w.detach(), "CostRegNet weight") for w in self.weight_list()]
        running, mode, momentum = _bn_call_args(self.bn_modules(), self.training)
        entry = "mvsn_costreg_forward_bn" if volume_dtype == torch.float32 else "mvsn_costreg_forward_f16"
        with torch.cuda.device(cost.device):
            _lib.check(getattr(lib, entry)(_lib.ptr_array(weights), _lib.ptr_array(running), mode, momentum,
                                           _lib.ptr(cost), D, Hp, Wp, _lib.ptr(vol), _lib.ptr(ws), ws_bytes,
                                           _lib.stream_ptr()), entry)
        return vol.permute(3, 0, 1, 2).unsqueeze(0)


class FrozenEncoderWarning(UserWarning):
    """MVSNet.forward was called under autograd with trainable encoder parameters (see its message)."""


class MVSNet(nn.Module):
    """Encoding-volume builder with the reference's call signature (models.py:771-932).  `.train()` / `.eval()` select
    batch-statistics or running-statistics BatchNorm exactly as for the reference module (every shipped caller runs
    `.train()` first, SURVEY.md F2; eval mode gives very different volumes with the shipped checkpoint, App. D)."""

    def __init__(self):
        super().__init__()
        self.feature = FeatureNet()
        self.cost_reg_2 = CostRegNet(32 + 9)
        self.N_importance = 0
        self.chunk = 1024

    def build_volume_costvar_img(self, imgs, feats, proj_mats, depth_values, pad=0):
        """models.py:839-893.  imgs [1,V,3,H,W], feats [1,V,32,h,w], proj_mats [1,V,3,4], depth_values [1,D]
        -> (img_feat [1,41,D,h',w'], in_masks [1,V,D,h',w'])."""
        lib = _lib.load()
        B, V, C, h, w = feats.shape
        if B != 1:
            raise RuntimeError("MVSNet: batch size must be 1 (as in every reference call site)")
        H, W = imgs.shape[-2:]
        D = depth_values.shape[-1]
        dev = feats.device
        imgs_c = _lib.dev_f32(imgs.reshape(V, 3, H, W), "imgs")
        feats_c = _lib.dev_f32(feats.reshape(V, C, h, w).detach(), "feats")
        proj_c = _lib.dev_f32(proj_mats.reshape(V, 3, 4).to(dev), "proj_mats")
        depth_c = _lib.dev_f32(depth_values.reshape(D).to(dev), "depth_values")
        hp, wp = h + 2 * pad, w + 2 * pad
        cost = torch.empty(1, 41, D, hp, wp, dtype=torch.float32, device=dev)
        masks = torch.empty(1, V, D, hp, wp, dtype=torch.float32, device=dev)
        ws_bytes = lib.mvsn_cost_volume_workspace_bytes(V, h, w)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.mvsn_build_cost_volume(_lib.ptr(imgs_c), _lib.ptr(feats_c), _lib.ptr(proj_c),
                                                  _lib.ptr(depth_c), V, H, W, D, int(pad), _lib.ptr(cost),
                                                  _lib.ptr(masks), _lib.ptr(ws), ws_bytes, _lib.stream_ptr()),
                       "mvsn_build_cost_volume")
        return cost, masks

    def forward(self, imgs, proj_mats, near_far, pad=0, return_color=False, lindisp=False, volume_dtype=torch.float32):
        """volume_dtype=torch.float16: the encoding volume is returned in fp16 (channels-last, half the bytes),
        bit-identical to .half() of the fp32 volume; the tensor-core render modes read it as it is."""
        if not imgs.is_cuda:
            raise RuntimeError("MVSNet: inputs must be CUDA tensors; mvsnerf_b200 has no CPU path")
        if torch.is_grad_enabled() and (imgs.requires_grad or any(p.requires_grad for p in self.parameters())):
            # train_mvs_nerf_pl.py:113 trains the encoder through this call; the kernels here are forward-only
            warnings.warn("mvsnerf_b200.MVSNet.forward runs forward-only CUDA kernels: the returned encoding volume "
                          "carries no autograd graph, so FeatureNet / CostRegNet receive no gradients (the encoder is "
                          "frozen). Call it under torch.no_grad() (as train_mvs_nerf_finetuning_pl.py:63 does) or "
                          "freeze the module to silence this.", FrozenEncoderWarning, stacklevel=2)
        B, V, _, H, W = imgs.shape
        feats = self.feature(imgs.reshape(B * V, 3, H, W))
        feats_l = feats.view(B, V, *feats.shape[1:])
        t = torch.linspace(0.0, 1.0, steps=N_DEPTH_PLANES, device=imgs.device, dtype=imgs.dtype)
        near, far = near_far
        if not lindisp:
            depth_values = near * (1.0 - t) + far * t
        else:
            depth_values = 1.0 / (1.0 / near * (1.0 - t) + 1.0 / far * t)
        depth_values = depth_values.unsqueeze(0)
        cost, in_masks = self.build_volume_costvar_img(imgs, feats_l, proj_mats, depth_values, pad=pad)
        if return_color:
            feats_l = torch.cat((cost[:, :V * 3].view(B, V, 3, *cost.shape[2:]), in_masks.unsqueeze(2)), dim=2)
        volume = self.cost_reg_2(cost, volume_dtype)
        return volume, feats_l, depth_values


class _RendererV0(nn.Module):
    """Parameter layout of Renderer_ours (models.py:145-222) for net_type 'v0'."""

    def __init__(self, D=6, W=128, input_ch=63, input_ch_views=3, input_ch_feat=20, skips=(4,)):
        super().__init__()
        if (D, W, input_ch, input_ch_views, input_ch_feat, tuple(skips)) != (6, 128, 63, 3, 20, (4,)):
            raise RuntimeError("the CUDA render kernel is built for the v0 network of ckpts/mvsnerf-v0.tar: "
                               "netdepth 6, netwidth 128, 63-ch positional encoding, 3-ch view dir, 20 features")
        self.skips = tuple(skips)
        self.pts_linears = nn.ModuleList(
            [nn.Linear(input_ch, W)] + [nn.Linear(W + input_ch if (i in self.skips) else W, W) for i in range(D - 1)])
        self.pts_bias = nn.Linear(input_ch_feat, W)
        self.views_linears = nn.ModuleList([nn.Linear(input_ch_views + W, W // 2)])
        self.feature_linear = nn.Linear(W, W)
        self.alpha_linear = nn.Linear(W, 1)
        self.rgb_linear = nn.Linear(W // 2, 3)

    def trunk(self, pts, feats):
        mod = self.pts_bias(feats)
        h = pts
        for i, layer in enumerate(self.pts_linears):
            h = F.relu(layer(h) * mod)
            if i in self.skips:
                h = torch.cat([pts, h], -1)
        return h

    def forward_alpha(self, x):
        pts, feats = x[..., :63], x[..., 63:]
        return torch.relu(self.alpha_linear(self.trunk(pts, feats)))

    def forward(self, x):
        pts, feats, dirs = x[..., :63], x[..., 63:83], x[..., 83:]
        h = self.trunk(pts, feats)
        sigma = torch.relu(self.alpha_linear(h))
        hv = F.relu(self.views_linears[0](torch.cat([self.feature_linear(h), dirs], -1)))
        return torch.cat([torch.sigmoid(self.rgb_linear(hv)), sigma], -1)


class MVSNeRF(nn.Module):
    """models.py:540-567.  `.nerf.*` parameter names as in network_fn_state_dict.  The PyTorch
    forward below exists for the non-hot-path callers (alpha-only queries); `rendering` never uses
    it -- it hands the parameters to the fused kernel."""

    def __init__(self, D=6, W=128, input_ch_pts=63, input_ch_views=3, input_ch_feat=20, skips=(4,), net_type="v0"):
        super().__init__()
        if net_type != "v0":
            raise RuntimeError(f"net_type {net_type!r}: only 'v0' (the shipped checkpoint) is implemented")
        self.nerf = _RendererV0(D, W, input_ch_pts, input_ch_views, input_ch_feat, skips)
        self._packed = {}

    def forward(self, x):
        return self.nerf(x)

    def forward_alpha(self, x):
        return self.nerf.forward_alpha(x)

    def ordered_params(self):
        n = self.nerf
        out = []
        for layer in n.pts_linears:
            out += [layer.weight, layer.bias]
        out += [n.pts_bias.weight, n.pts_bias.bias, n.views_linears[0].weight, n.views_linears[0].bias,
                n.feature_linear.weight, n.feature_linear.bias, n.alpha_linear.weight, n.alpha_linear.bias,
                n.rgb_linear.weight, n.rgb_linear.bias]
        return out

    def packed(self, mode=_lib.MLP_FP32):
        """Kernel-layout weight image; re-packed whenever a parameter was modified in place."""
        lib = _lib.load()
        params = self.ordered_params()
        dev = params[0].device
        if not params[0].is_cuda:
            raise RuntimeError("network_fn must live on a CUDA device; mvsnerf_b200 has no CPU path")
        key = (mode, dev, tuple(p._version for p in params), tuple(p.data_ptr() for p in params))
        hit = self._packed.get(mode)
        if hit is not None and hit[0] == key:
            return hit[1]
        nbytes = lib.mvsn_mlp_packed_bytes(mode)
        if nbytes == 0:
            raise RuntimeError(f"MLP mode {mode} is not available in this build of libmvsnerf_b200")
        buf = hit[1] if hit is not None and hit[1].numel() == nbytes and hit[1].device == dev else \
            torch.empty(nbytes, dtype=torch.uint8, device=dev)
        srcs = [_lib.dev_f32(p.detach(), "MLP parameter") for p in params]
        with torch.cuda.device(dev):
            _lib.check(lib.mvsn_mlp_pack(_lib.ptr_array(srcs), mode, _lib.ptr(buf), nbytes, _lib.stream_ptr()),
                       "mvsn_mlp_pack")
        self._packed[mode] = (key, buf)
        return buf


class RefVolume(nn.Module):
    """models.py:935-950: the encoding volume as a parameter (per-scene fine-tuning)."""

    def __init__(self, volume):
        super().__init__()
        self.feat_volume = nn.Parameter(volume)

    def forward(self, ray_coordinate_ref):
        H, W = ray_coordinate_ref.shape[-3:-1]
        grid = ray_coordinate_ref.view(-1, 1, H, W, 3).to(self.feat_volume.device) * 2 - 1.0
        f = F.grid_sample(self.feat_volume, grid, align_corners=True, mode="bilinear")
        return f[:, :, 0].permute(2, 3, 0, 1).squeeze()


# --------------------------------------------------------------------------------------------
# scene-constant device state (packed images, channels-last volume), cached per tensor version
# --------------------------------------------------------------------------------------------
_cache = {}


cache_stats = {"hit": 0, "miss": 0}


def _cached(kind, t, build):
    """One entry per kind, keyed on the IDENTITY of the caller's tensor object (held by weakref)
    and its in-place version counter -- never on data_ptr, which the caching allocator recycles.
    `t` must be the object the CALLER holds (a Parameter, a checkpoint tensor), not a view made here."""
    hit = _cache.get(kind)
    if hit is not None and hit[0]() is t and hit[1] == t._version:
        cache_stats["hit"] += 1
        return hit[2]
    cache_stats["miss"] += 1
    val = build()
    _cache[kind] = (weakref.ref(t), t._version, val)
    return val


def clear_cache():
    _cache.clear()


def _volume_channels_last(volume_feature, half_ok=False):
    """Accepts a tensor [1,8,D,Hp,Wp] (any strides) or a RefVolume; returns ([D,Hp,Wp,8] fp32, dims).  With `half_ok`
    (a tensor-core render), a float16 volume is returned as an fp16 image instead (MVSN_VOLUME_F16)."""
    owner = volume_feature.feat_volume if isinstance(volume_feature, nn.Module) else volume_feature
    vol = owner.detach()          # a NEW tensor object every call: the cache below is keyed on `owner`
    if vol.dim() != 5 or vol.shape[0] != 1 or vol.shape[1] != 8:
        raise RuntimeError(f"encoding volume must be [1,8,D,H,W], got {tuple(vol.shape)}")
    if not vol.is_cuda:
        raise RuntimeError("encoding volume must be a CUDA tensor; mvsnerf_b200 has no CPU path")
    _, _, D, Hp, Wp = vol.shape
    cl = vol[0].permute(1, 2, 3, 0)
    if half_ok and vol.dtype == torch.float16:
        if cl.is_contiguous():
            return cl, (D, Hp, Wp)                     # MVSNet.forward(volume_dtype=float16) or .half() of it: zero-copy

        def build_f16():
            lib = _lib.load()
            src = vol[0].contiguous()                  # planar [8,D,Hp,Wp]: a view for a contiguous volume
            dst = torch.empty(D, Hp, Wp, 8, dtype=torch.float16, device=vol.device)
            with torch.cuda.device(vol.device):
                _lib.check(lib.mvsn_volume_to_half(_lib.ptr(src), 1, 1, D, Hp, Wp, _lib.ptr(dst), _lib.stream_ptr()),
                           "mvsn_volume_to_half")
            return dst

        return _cached("volume_f16", owner, build_f16), (D, Hp, Wp)
    if vol.dtype == torch.float32 and cl.is_contiguous():
        return cl, (D, Hp, Wp)                         # MVSNet.forward output: zero-copy

    def build():
        lib = _lib.load()
        src = _lib.dev_f32(vol[0], "volume")
        dst = torch.empty(D, Hp, Wp, 8, dtype=torch.float32, device=vol.device)
        with torch.cuda.device(vol.device):
            _lib.check(lib.mvsn_volume_to_channels_last(_lib.ptr(src), D, Hp, Wp, _lib.ptr(dst), _lib.stream_ptr()),
                       "mvsn_volume_to_channels_last")
        return dst

    return _cached("volume", owner, build), (D, Hp, Wp)


def _images_packed(imgs):
    """imgs [1,V,3,H,W] un-normalised -> [V,H,W,4]."""
    if imgs.dim() != 5 or imgs.shape[0] != 1 or imgs.shape[2] != 3:
        raise RuntimeError(f"imgs must be [1,V,3,H,W], got {tuple(imgs.shape)}")
    if not imgs.is_cuda:
        raise RuntimeError("imgs must be a CUDA tensor; mvsnerf_b200 has no CPU path")
    _, V, _, H, W = imgs.shape

    def build():
        lib = _lib.load()
        src = _lib.dev_f32(imgs[0].detach(), "imgs")
        dst = torch.empty(V, H, W, 4, dtype=torch.float32, device=imgs.device)
        with torch.cuda.device(imgs.device):
            _lib.check(lib.mvsn_pack_images(_lib.ptr(src), V, H, W, _lib.ptr(dst), _lib.stream_ptr()),
                       "mvsn_pack_images")
        return dst

    return _cached("imgs", imgs, build), (V, H, W)


def _make_scene(pose_ref, volume_feature, imgs, network_fn, white_bkgd, mode, half_ok=False, half_fp32=False):
    """half_ok: a forward render that may read a float16 volume as fp16 (tensor-core modes only); otherwise a half
    volume is upcast to a cached fp32 image.  half_fp32: MLP_FP32 reads it as fp16 too (mvsn_build_density)."""
    vol, (D, Hp, Wp) = _volume_channels_last(volume_feature, half_ok and (mode != _lib.MLP_FP32 or half_fp32))
    im, (V, H, W) = _images_packed(imgs)
    if V != 3:
        raise RuntimeError(f"{V} source views: the v0 network takes exactly 3 (feat_dim = 8 + 3*4)")
    sc = _lib.RenderScene()
    sc.volume_dhwc, sc.D, sc.Hp, sc.Wp = vol.data_ptr(), D, Hp, Wp
    sc.imgs_hwc4, sc.V, sc.H, sc.W = im.data_ptr(), V, H, W
    w2cs = _lib.dev_f32(pose_ref["w2cs"].detach(), "pose_ref['w2cs']")               # [V,4,4]
    intr = _lib.dev_f32(pose_ref["intrinsics"].detach(), "pose_ref['intrinsics']")   # [V,3,3]
    if tuple(w2cs.shape) != (3, 4, 4) or tuple(intr.shape) != (3, 3, 3):
        raise RuntimeError(f"pose_ref: expected w2cs [3,4,4] and intrinsics [3,3,3], got "
                           f"{tuple(w2cs.shape)} and {tuple(intr.shape)}")
    sc.w2cs, sc.intrinsics = w2cs.data_ptr(), intr.data_ptr()
    packed = network_fn.packed(mode)
    if vol.dtype == torch.float16:
        mode |= _lib.VOLUME_F16
    sc.mlp_packed, sc.mlp_mode, sc.white_bkgd = packed.data_ptr(), mode, int(bool(white_bkgd))
    keep = (vol, im, packed, w2cs, intr)          # keep the device buffers alive for the duration of the call
    return sc, keep


# Default arithmetic of `rendering` / `render_rays`: the fp32-grade tensor-core mode (2-term fp16 operand split,
# RGB Linf 1.2e-5 vs the reference on every pixel of the 512x640 config -- the same as the FFMA kernel, several
# times faster).  MLP_FP32 (FFMA) and MLP_TC_HALF / MLP_TC_PAIR (5e-3 tier) are selected with `mlp_mode=`.
DEFAULT_MLP_MODE = _lib.MLP_TC_SPLIT


def rendering(args, pose_ref, rays_pts, rays_ndc, depth_candidates, rays_o, rays_dir,
              volume_feature=None, imgs=None, network_fn=None, img_feat=None, network_query_fn=None,
              white_bkgd=False, **kwargs):
    """Drop-in for renderer.rendering (renderer.py:138-165).  Returns
    (rgb_map [N,3], input_feat [N,S,20], weights [N,S], depth_map [N], alpha [N,S], {}).

    Extra keyword arguments the reference's callers pass (perturb, N_importance, network_fine,
    use_viewdirs, raw_noise_std, NDC_local) are accepted and ignored, as the reference does.
    `mlp_mode=` selects the GEMM arithmetic (default: DEFAULT_MLP_MODE, the fp32-grade tensor mode); `want_aux=False` skips the three
    per-sample outputs (they are returned as None).  Under autograd, `grad_mode=` selects the arithmetic of the backward's
    GEMMs (see render_backward; default MLP_FP32).

    `t_stop=` (a float >= 0, tensor-core mlp_mode; None, the default, changes nothing): early ray termination
    (mvsn_render_samples_stop) -- a group of up to 32 neighbouring rays stops two tiles after every ray in it has
    transmittance < t_stop, so each channel of rgb differs from the full render by less than t_stop and depth by less
    than t_stop * max(z) (t_stop = 0: bit-identical).  The samples behind are not computed, so the three per-sample
    outputs (input_feat, weights, alpha) are returned as None.  `tiles_done=`: an optional CUDA int64 tensor [1] the
    number of computed 64-sample tiles is added to.  Under autograd t_stop must lie in [0, 1]; the backward is
    render_backward(..., t_stop=t_stop) with the rgb and depth cotangents: each ray back-propagates the prefix of samples
    whose transmittance in front of them is >= t_stop.  create_nerf_mvs puts `t_stop` into the render kwargs when the
    caller's `args` has one."""
    if pose_ref is None or img_feat is not None or getattr(args, "use_color_volume", False):
        raise RuntimeError("rendering: only the pose_ref / image-gather branch of the reference is implemented "
                           "(use_color_volume=False, img_feat=None) -- the branch every shipped config uses")
    mode = kwargs.pop("mlp_mode", DEFAULT_MLP_MODE)
    want_aux = kwargs.pop("want_aux", True)
    grad_mode = kwargs.pop("grad_mode", _lib.MLP_FP32)
    t_stop = kwargs.pop("t_stop", None)
    tiles_done = kwargs.pop("tiles_done", None)
    _check_grad_mode(grad_mode)
    if t_stop is not None:
        t_stop = float(t_stop)
        if not t_stop >= 0.0:
            raise RuntimeError(f"rendering: t_stop={t_stop} must be >= 0")
        if mode == _lib.MLP_FP32:
            raise RuntimeError("rendering: t_stop needs a tensor-core mlp_mode (MLP_TC_HALF / TC_PAIR / TC_SPLIT)")
        _check_counter(tiles_done, "rendering", "tiles_done", torch.int64, 1, rays_pts.device)
    elif tiles_done is not None:
        raise RuntimeError("rendering: tiles_done needs t_stop")
    N, S = rays_pts.shape[:2]
    z = depth_candidates.expand(N, S) if depth_candidates.shape != (N, S) else depth_candidates
    vol_t = volume_feature.feat_volume if isinstance(volume_feature, nn.Module) else volume_feature
    if torch.is_grad_enabled() and (vol_t.requires_grad or any(p.requires_grad for p in network_fn.parameters())):
        # training step (fine-tuning, train_mvs_nerf_finetuning_pl.py:164): same kernel forward, gradients for
        # the MLP parameters and the encoding volume (see _RenderSamplesFn)
        params = network_fn.ordered_params()
        if t_stop is not None and t_stop > 1.0:
            raise RuntimeError(f"rendering: t_stop={t_stop} must be in [0, 1] under autograd (see render_backward)")
        stop = () if t_stop is None else ((t_stop, tiles_done),)
        rgb, feat, weights, depth, alpha = _RenderSamplesFn.apply(
            rays_pts, rays_ndc, z, rays_dir, vol_t, imgs, pose_ref["w2cs"], pose_ref["intrinsics"],
            bool(white_bkgd), mode, network_fn, volume_feature, (grad_mode,) + stop, *params)
        return rgb, feat, weights, depth, alpha, {}
    rgb, feat, weights, depth, alpha = _render_samples_kernel(
        pose_ref, rays_pts, rays_ndc, z, rays_dir, volume_feature, imgs, network_fn, white_bkgd, mode, want_aux,
        half_ok=True, t_stop=t_stop, tiles_done=tiles_done)
    return rgb, feat, weights, depth, alpha, {}


def _check_counter(t, who, name, dtype, n, device):
    """An optional output counter (live_samples / tiles_done): a contiguous CUDA `dtype` tensor of >= n elements on
    `device`."""
    if t is not None and (not t.is_cuda or t.device != device or t.dtype != dtype or t.numel() < n
                          or not t.is_contiguous()):
        raise RuntimeError(f"{who}: {name} must be a contiguous CUDA {dtype} tensor of >= {n} elements on the input's "
                           f"device ({device})")


def _render_samples_kernel(pose_ref, rays_pts, rays_ndc, z, rays_dir, volume_feature, imgs, network_fn, white_bkgd,
                           mode, want_aux=True, half_ok=False, t_stop=None, tiles_done=None):
    """One mvsn_render_samples launch (no autograd graph); half_ok: see _make_scene.  With `t_stop`: one
    mvsn_render_samples_stop launch, and the per-sample outputs are None."""
    lib = _lib.load()
    N, S = rays_pts.shape[:2]
    dev = rays_pts.device
    pts = _lib.dev_f32(rays_pts.detach(), "rays_pts")
    ndc = _lib.dev_f32(rays_ndc.detach(), "rays_ndc")
    z = _lib.dev_f32(z.detach(), "depth_candidates")
    dirs = _lib.dev_f32(rays_dir.detach(), "rays_dir")
    sc, keep = _make_scene(pose_ref, volume_feature, imgs, network_fn, white_bkgd, mode, half_ok)
    rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
    depth = torch.empty(N, dtype=torch.float32, device=dev)
    feat = weights = alpha = None
    if t_stop is not None:
        with torch.cuda.device(dev):
            _lib.check(lib.mvsn_render_samples_stop(C.byref(sc), _lib.ptr(pts), _lib.ptr(ndc), _lib.ptr(z), _lib.ptr(dirs),
                                                    N, S, t_stop, _lib.ptr(rgb), _lib.ptr(depth), _lib.ptr(tiles_done),
                                                    _lib.stream_ptr()), "mvsn_render_samples_stop")
        del keep
        return rgb, feat, weights, depth, alpha
    if want_aux:
        feat = torch.empty(N, S, 20, dtype=torch.float32, device=dev)
        weights = torch.empty(N, S, dtype=torch.float32, device=dev)
        alpha = torch.empty(N, S, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.mvsn_render_samples(C.byref(sc), _lib.ptr(pts), _lib.ptr(ndc), _lib.ptr(z), _lib.ptr(dirs),
                                           N, S, _lib.ptr(rgb), _lib.ptr(depth), _lib.ptr(weights), _lib.ptr(alpha),
                                           _lib.ptr(feat), _lib.stream_ptr()), "mvsn_render_samples")
    del keep
    return rgb, feat, weights, depth, alpha


def _render_samples_torch(pts, ndc, z, rays_dir, vol, imgs, w2cs, intrinsics, nerf, white_bkgd):
    """Differentiable PyTorch statement of renderer.rendering (renderer.py:138-165) -- used ONLY inside
    _RenderSamplesFn.backward to obtain gradients; forward values always come from the CUDA kernel."""
    N, S = pts.shape[:2]
    _, V, _, H, W = imgs.shape
    grid = (ndc * 2 - 1.0).view(1, 1, N, S, 3)
    vfeat = F.grid_sample(vol, grid, mode="bilinear", padding_mode="zeros", align_corners=True)[0, :, 0].permute(1, 2, 0)
    inv_scale = torch.tensor([W - 1.0, H - 1.0], device=pts.device)
    cols = []
    for v in range(V):                                                           # utils.py:300-332
        cam = pts.reshape(-1, 3) @ w2cs[v, :3, :3].t() + w2cs[v, :3, 3].view(1, 3)
        pix = cam @ intrinsics[v].t()
        g = ((pix[:, :2] / pix[:, 2:3] / inv_scale) * 2 - 1.0).view(1, N, S, 2)
        c = F.grid_sample(imgs[0, v:v + 1], g, mode="bilinear", padding_mode="border", align_corners=True)[0].permute(1, 2, 0)
        m = ((g[0] > -1.0) & (g[0] < 1.0)).all(-1, keepdim=True).to(c.dtype)
        cols += [c, m]
    feat = torch.cat([vfeat] + cols, -1)
    d = rays_dir / rays_dir.norm(dim=-1, keepdim=True)
    d = d @ w2cs[0, :3, :3].t()                                                  # renderer.py:111-122
    raw = nerf(torch.cat([_embed(ndc), feat, d[:, None].expand(-1, S, -1)], -1))
    alpha = 1.0 - torch.exp(-raw[..., 3])                                        # renderer.py:18-26
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    weights = alpha * trans
    rgb = (weights.unsqueeze(-1) * raw[..., :3]).sum(-2)
    depth = (weights * z).sum(-1)
    if white_bkgd:
        rgb = rgb + (1.0 - weights.sum(-1, keepdim=True))
    return rgb, feat, weights, depth, alpha


class _RenderSamplesFn(torch.autograd.Function):
    """Training-step form of `rendering` (SURVEY.md 8(f) row 2).

    forward: the fused CUDA kernel, exactly as in inference (no graph, nothing per-sample kept).
    backward: gradients w.r.t. the 22 MLP tensors and the encoding volume.  With N_samples <= 128 (and
    BACKWARD_IMPL == "kernel") they come from the backward kernel (csrc/render_bwd.cu: forward recompute on the
    fp32 render kernel's own forward tile, MLP dgrad/wgrad in the arithmetic `grad_mode` selects, trilinear scatter
    into the volume gradient; bit-reproducible under torch.use_deterministic_algorithms(True), see render_backward).
    Otherwise the chunk is re-evaluated with PyTorch ops under autograd (_render_samples_torch); activation memory then
    exists only during backward.

    `how` = (grad_mode,) or, with early ray termination, (grad_mode, (t_stop, tiles_done)): the forward is then
    mvsn_render_samples_stop (the per-sample outputs are None) and the backward render_backward(..., t_stop=t_stop)
    with the rgb and depth cotangents (the kernel path only; a non-zero per-sample cotangent raises)."""

    @staticmethod
    def forward(ctx, pts, ndc, z, rays_dir, vol, imgs, w2cs, intrinsics, white_bkgd, mode, network_fn, volume_feature,
                how, *params):
        pose = {"w2cs": w2cs, "intrinsics": intrinsics}
        grad_mode, stop = how[0], (how[1] if len(how) > 1 else (None, None))
        kw = {} if stop[0] is None else {"t_stop": stop[0], "tiles_done": stop[1]}
        out = _render_samples_kernel(pose, pts, ndc, z, rays_dir, volume_feature, imgs, network_fn, white_bkgd, mode, **kw)
        ctx.save_for_backward(pts, ndc, z, rays_dir, vol, imgs, w2cs, intrinsics, *params)
        ctx.white_bkgd, ctx.network_fn, ctx.volume_feature = white_bkgd, network_fn, volume_feature
        ctx.grad_mode, ctx.t_stop = grad_mode, stop[0]
        return out

    @staticmethod
    def backward(ctx, g_rgb, g_feat, g_weights, g_depth, g_alpha):
        pts, ndc, z, rays_dir, vol, imgs, w2cs, intrinsics, *params = ctx.saved_tensors
        S = pts.shape[1]
        if ctx.t_stop is not None:
            # early ray termination: the truncated render of the kernel backward, which has no per-sample outputs
            if any(g is not None and bool(g.any()) for g in (g_feat, g_weights, g_alpha)):
                raise RuntimeError("rendering with t_stop: input_feat / weights / alpha are not computed for dead samples "
                                   "and take no cotangent")
            if S > 128 or BACKWARD_IMPL != "kernel":
                raise RuntimeError(f"rendering with t_stop: the backward kernel takes N_samples <= 128 (got {S})")
        if S <= 128 and BACKWARD_IMPL == "kernel":
            # the hand-written backward kernel (csrc/render_bwd.cu): recompute + dgrad/wgrad + volume scatter
            need_vol = ctx.needs_input_grad[4]
            grads = {"rgb": g_rgb, "depth": g_depth}
            if ctx.t_stop is None:
                grads.update(weights=g_weights, alpha=g_alpha, input_feat=g_feat)
            g_params, dvol, _, _ = render_backward(
                {"w2cs": w2cs, "intrinsics": intrinsics}, pts, ndc, z, rays_dir, ctx.volume_feature, imgs, ctx.network_fn,
                ctx.white_bkgd, grads=grads, want_volume_grad=need_vol, grad_mode=ctx.grad_mode, t_stop=ctx.t_stop)
            g_vol = dvol.permute(3, 0, 1, 2).unsqueeze(0) if need_vol else None
            g_params = [g if need else None for g, need in zip(g_params, ctx.needs_input_grad[13:])]
            return (None, None, None, None, g_vol, None, None, None, None, None, None, None, None, *g_params)
        with torch.enable_grad():
            vol_g = vol.detach().requires_grad_(ctx.needs_input_grad[4])
            # evaluate through a functional copy of the module so the user's parameters are not touched
            leaves = [p.detach().requires_grad_(need) for p, need in zip(params, ctx.needs_input_grad[13:])]
            names = [n for n, _ in _ordered_named_params(ctx.network_fn)]
            nerf = lambda x: torch.func.functional_call(ctx.network_fn, dict(zip(names, leaves)), (x,))
            outs = _render_samples_torch(pts.detach(), ndc.detach(), z.detach(), rays_dir.detach(), vol_g, imgs.detach(),
                                         w2cs.detach(), intrinsics.detach(), nerf, ctx.white_bkgd)
            pairs = [(o, g) for o, g in zip(outs, (g_rgb, g_feat, g_weights, g_depth, g_alpha))
                     if g is not None and o.requires_grad]
            wrt = [t for t in [vol_g] + leaves if t.requires_grad]
            grads = torch.autograd.grad([o for o, _ in pairs], wrt, [g for _, g in pairs], allow_unused=True) if wrt and pairs else []
        it = iter(grads)
        g_vol = next(it) if vol_g.requires_grad and grads else None
        g_params = [next(it) if (leaf.requires_grad and grads) else None for leaf in leaves]
        return (None, None, None, None, g_vol, None, None, None, None, None, None, None, None, *g_params)


# "kernel": csrc/render_bwd.cu (N_samples <= 128); "torch": the PyTorch-recompute backward above (kept as the
# independent statement the gradient tests compare against, and for N_samples > 128)
BACKWARD_IMPL = "kernel"
_bwd_workspace = {}


def _check_grad_mode(grad_mode, rays=False):
    """`rays`: the entry marches its samples from rays (render_backward_rays, FineTuner.step_rays), the only ones that
    take GRAD_TC_FULL."""
    if grad_mode == _lib.GRAD_TC_FULL and not rays:
        raise RuntimeError("grad_mode GRAD_TC_FULL (the forward recompute on tensor cores too) is taken by "
                           "FineTuner.step_rays and render_backward_rays only; the samples entries (FineTuner.step, "
                           "render_backward, rendering under autograd) run MLP_FP32 or MLP_TC_HALF")
    if grad_mode not in (_lib.MLP_FP32, _lib.MLP_TC_HALF, _lib.GRAD_TC_FULL):
        raise RuntimeError(f"grad_mode {grad_mode!r}: the backward's GEMMs run in MLP_FP32 (FFMA) or MLP_TC_HALF "
                           "(wgmma, fp16 operands with per-tile power-of-two scales, fp32 accumulation)")


def _backward(who, rays, inputs, dev, N, S, pose_ref, volume_feature, imgs, network_fn, white_bkgd, grads, target_rgb,
              n_total, want_volume_grad, grad_volume, grad_mlp, want_forward, loss_out, grad_mode, t_stop, live_samples,
              tiles_done):
    """One launch of a backward C entry over N rays x S samples on `dev`: render_backward (`rays` False) or
    render_backward_rays (`who`).  Every argument is checked before `inputs()` prepares the entry's own: it returns the
    C arguments between the weights and N, and the objects they point into."""
    _check_grad_mode(grad_mode, rays)
    if t_stop is not None:
        t_stop = float(t_stop)
        if not 0.0 <= t_stop <= 1.0:
            raise RuntimeError(f"{who}: t_stop={t_stop} must be in [0, 1]")
        if grads is not None and any(grads.get(k) is not None for k in ("weights", "alpha", "input_feat")):
            raise RuntimeError(f"{who}: t_stop takes no per-sample cotangents (weights / alpha / input_feat):"
                               " dead samples have none")
        _check_counter(live_samples, who, "live_samples", torch.int32, N, dev)
        _check_counter(tiles_done, who, "tiles_done", torch.int64, 3, dev)
    elif live_samples is not None or tiles_done is not None:
        raise RuntimeError(f"{who}: live_samples / tiles_done need t_stop")
    lib = _lib.load()
    args, held_inputs = inputs()
    sc, keep = _make_scene(pose_ref, volume_feature, imgs, network_fn, white_bkgd, _lib.MLP_FP32)
    params = [_lib.dev_f32(p.detach(), "MLP parameter") for p in network_fn.ordered_params()]
    if grad_mlp is None:
        grad_mlp = [torch.empty_like(p) for p in params]
    if want_volume_grad and grad_volume is None:
        grad_volume = torch.zeros(sc.D, sc.Hp, sc.Wp, 8, dtype=torch.float32, device=dev)
    g, held, rgb, depth = _render_grads(N, S, dev, grads, target_rgb, n_total, want_forward, loss_out)
    det = torch.are_deterministic_algorithms_enabled()
    dims = (sc.D, sc.Hp, sc.Wp) if want_volume_grad else (0, 0, 0)
    # mvsn_render_backward_rays[_stop] and mvsn_render_backward_stop take (grad_mode, deterministic[, t_stop]); the
    # other samples entries are named by their summation order, and by their grad mode unless deterministic
    if rays or t_stop is not None:
        name = "mvsn_render_backward" + ("_rays" if rays else "") + ("_stop" if t_stop is not None else "")
        modes = (int(grad_mode), int(det)) + (() if t_stop is None else (t_stop,))
        need = getattr(lib, name + "_workspace_bytes")(N, S, *dims, int(grad_mode), int(det))
    elif det:
        name, modes = "mvsn_render_backward_deterministic", (int(grad_mode),)
        need = lib.mvsn_render_backward_deterministic_workspace_bytes(N, S, *dims, int(grad_mode))
    else:
        name = "mvsn_render_backward_tc" if grad_mode == _lib.MLP_TC_HALF else "mvsn_render_backward"
        modes, need = (), getattr(lib, name + "_workspace_bytes")(N, S)
    if need == 0:
        raise RuntimeError(f"{who}: unsupported shape N={N}, N_samples={S} (N_samples <= 128)")
    ws = _bwd_workspace.get(dev)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        _bwd_workspace[dev] = ws
    counters = () if t_stop is None else (_lib.ptr(live_samples), _lib.ptr(tiles_done))
    with torch.cuda.device(dev):
        _lib.check(getattr(lib, name)(C.byref(sc), _lib.ptr_array(params), *args, N, S, *modes, C.byref(g),
                                      _lib.ptr_array(grad_mlp), _lib.ptr(grad_volume) if want_volume_grad else None,
                                      *counters, _lib.ptr(ws), need, _lib.stream_ptr()), name)
    del keep, held, held_inputs
    return grad_mlp, (grad_volume if want_volume_grad else None), rgb, depth


def render_backward(pose_ref, rays_pts, rays_ndc, z_vals, rays_dir, volume_feature, imgs, network_fn, white_bkgd=False,
                    grads=None, target_rgb=None, n_total=None, want_volume_grad=True, grad_volume=None, grad_mlp=None,
                    want_forward=False, loss_out=None, grad_mode=_lib.MLP_FP32, t_stop=None, live_samples=None,
                    tiles_done=None):
    """One mvsn_render_backward launch (grad_mode=MLP_FP32: fp32 FFMA GEMMs) or mvsn_render_backward_tc launch
    (grad_mode=MLP_TC_HALF: the dgrad / wgrad GEMMs on tensor cores with fp16 operands, fp32 accumulation; the forward
    recompute, and so rgb / depth / the loss, are the same fp32 tile and bit-identical).  Either `grads` (dict with 'rgb' and optionally 'depth', 'weights', 'alpha',
    'input_feat': d loss / d output of `rendering`) or `target_rgb` [N,3] (img2mse formed in the kernel, normalised by
    3 * n_total).  Returns (grad_mlp[22] in ordered_params() order, grad_volume [D,Hp,Wp,8] channels-last or None,
    rgb [N,3] or None, depth [N] or None).  `grad_volume` (accumulated into) and `grad_mlp` (overwritten) may be passed
    to reuse buffers.

    With torch.use_deterministic_algorithms(True) in effect at call time the launch is
    mvsn_render_backward_deterministic instead (same grad_mode): the volume gradient and the fused loss are summed in
    a fixed order, so every output is bit-reproducible; otherwise they are summed with float atomics.

    `t_stop` (a float in [0, 1]): early ray termination (mvsn_render_backward_stop, same grad_mode and summation-order
    dispatch) -- each ray keeps the prefix of samples whose transmittance in front of them is >= t_stop, and the step
    renders, forms the loss of and exactly differentiates that truncated render; each channel differs from the full
    render by less than t_stop (t_stop = 0: bit-identical to t_stop=None).  Per-sample cotangents (`grads` 'weights',
    'alpha', 'input_feat') are rejected with it.  `live_samples`: an optional CUDA int32 tensor [N] that receives each
    ray's number of kept samples; `tiles_done`: an optional CUDA int64 tensor [3] the counts of tiles back-propagated
    immediately, deferred and packed are added to."""
    N, S = rays_pts.shape[:2]

    def inputs():
        pts = _lib.dev_f32(rays_pts.detach(), "rays_pts")
        ndc = _lib.dev_f32(rays_ndc.detach(), "rays_ndc")
        z = _lib.dev_f32((z_vals.expand(N, S) if z_vals.shape != (N, S) else z_vals).detach(), "depth_candidates")
        dirs = _lib.dev_f32(rays_dir.detach(), "rays_dir")
        return (_lib.ptr(pts), _lib.ptr(ndc), _lib.ptr(z), _lib.ptr(dirs)), (pts, ndc, z, dirs)
    return _backward("render_backward", False, inputs, rays_pts.device, N, S, pose_ref, volume_feature, imgs, network_fn,
                     white_bkgd, grads, target_rgb, n_total, want_volume_grad, grad_volume, grad_mlp, want_forward,
                     loss_out, grad_mode, t_stop, live_samples, tiles_done)


def _render_grads(N, S, dev, grads, target_rgb, n_total, want_forward, loss_out):
    """The lib.RenderGrads of a backward launch over N rays x S samples: the cotangents (`grads`) or the fused loss
    (`target_rgb`, normalised by 3 * n_total), and the optional forward / loss outputs.  Returns (g, the device tensors
    g points into, rgb [N,3] or None, depth [N] or None)."""
    g = _lib.RenderGrads()
    held = []

    def opt(t, shape, name):
        if t is None:
            return None
        t = _lib.dev_f32(t.detach(), name)
        if tuple(t.shape) != tuple(shape):
            t = t.expand(shape).contiguous()
        held.append(t)
        return t.data_ptr()
    if target_rgb is not None:
        g.target_rgb = opt(target_rgb, (N, 3), "target_rgb")
        g.loss_scale = 1.0 / (3.0 * float(N if n_total is None else n_total))
    else:
        if grads is None or grads.get("rgb") is None:
            grads = dict(grads or {})
            grads["rgb"] = torch.zeros(N, 3, dtype=torch.float32, device=dev)
        g.rgb = opt(grads["rgb"], (N, 3), "grad rgb")
    if grads is not None:
        g.depth = opt(grads.get("depth"), (N,), "grad depth")
        g.weights = opt(grads.get("weights"), (N, S), "grad weights")
        g.alpha = opt(grads.get("alpha"), (N, S), "grad alpha")
        g.input_feat = opt(grads.get("input_feat"), (N, S, 20), "grad input_feat")
    rgb = depth = None
    if want_forward:
        rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
        g.rgb_out, g.depth_out = rgb.data_ptr(), depth.data_ptr()
    if loss_out is not None:
        g.loss_out = loss_out.data_ptr()
    return g, held, rgb, depth


def _tsteps_of(S, dev):
    """torch.linspace(0, 1, S) on `dev` (data/ray_utils.py:175), cached: the t_steps of the in-kernel ray march."""
    tk = (S, dev)
    if tk not in _tsteps:
        _tsteps[tk] = torch.linspace(0, 1, S, device=dev)
    return _tsteps[tk]


def render_backward_rays(rays, volume_feature, imgs, pose_ref, network_fn, near_far, pad, N_samples=128, lindisp=False,
                         jitter=None, white_bkgd=False, grads=None, target_rgb=None, n_total=None, want_volume_grad=True,
                         grad_volume=None, grad_mlp=None, want_forward=False, loss_out=None, grad_mode=_lib.MLP_FP32,
                         t_stop=None, live_samples=None, tiles_done=None):
    """render_backward straight from rays [N,8] = (o, d, near, far): one mvsn_render_backward_rays launch, whose kernel
    also does ray_marcher and get_ndc_coordinate (data/ray_utils.py:152-197, utils.py:112-146) for the reference camera.
    `near_far` / `pad` / `N_samples` / `lindisp` as in render_rays.  `jitter` [N, N_samples] = perturb * u, the uniform
    draw ray_marcher makes with perturb > 0: sample s then lies at lower + (upper - lower) * jitter between the
    midpoints of its neighbours' depths, rounded as ray_marcher rounds it; None marches exactly render_rays' depths.
    Everything else, the return value and the grad_mode / torch.use_deterministic_algorithms dispatch are as in
    render_backward (the depth the `grads` dict differentiates is the jittered one).

    `t_stop` (a float in [0, 1]): early ray termination (mvsn_render_backward_rays_stop) -- each ray keeps the prefix of
    samples whose transmittance in front of them is >= t_stop, and the step renders, forms the loss of and exactly
    differentiates that truncated render; each channel differs from the full render by less than t_stop (t_stop = 0:
    bit-identical to t_stop=None).  Per-sample cotangents (`grads` 'weights', 'alpha', 'input_feat') are rejected with
    it.  `live_samples`: an optional CUDA int32 tensor [N] that receives each ray's number of kept samples;
    `tiles_done`: an optional CUDA int64 tensor [3] the counts of tiles back-propagated immediately, deferred and packed
    are added to.

    grad_mode=GRAD_TC_FULL: MLP_TC_HALF's backward, and the forward recompute's MLP on tensor cores too (fp16 operands,
    a power-of-two scale per sample row, fp32 accumulation; see MVSN_GRAD_TC_FULL in include/mvsnerf_b200.h).  rgb,
    depth and the loss are then that recompute's, within the 5e-3 tier of MLP_FP32."""
    N, S = rays.shape[0], int(N_samples)

    def inputs():
        r = _lib.dev_f32(rays.detach(), "rays")
        j = None if jitter is None else _lib.dev_f32(jitter.detach(), "jitter")
        if j is not None and tuple(j.shape) != (N, S):
            raise RuntimeError(f"render_backward_rays: jitter must be [{N}, {S}], got {tuple(j.shape)}")
        rp = _lib.RayParams(float(near_far[0]), float(near_far[1]), float(pad), int(bool(lindisp)))
        return (C.byref(rp), _lib.ptr(r), _lib.ptr(_tsteps_of(S, r.device)), _lib.ptr(j)), (rp, r, j)
    return _backward("render_backward_rays", True, inputs, rays.device, N, S, pose_ref, volume_feature, imgs, network_fn,
                     white_bkgd, grads, target_rgb, n_total, want_volume_grad, grad_volume, grad_mlp, want_forward,
                     loss_out, grad_mode, t_stop, live_samples, tiles_done)


class FineTuner:
    """The reference's per-scene fine-tuning step (train_mvs_nerf_finetuning_pl.py:140-189: rendering -> img2mse ->
    Adam over the MLP and RefVolume.feat_volume) as four launches and no autograd graph:

        mvsn_mlp_pack (fp32 image) -> mvsn_render_backward (forward recompute + loss + all gradients)
        -> mvsn_adam_step (22 MLP tensors) -> mvsn_adam_step_volume (volume; also zeroes its gradient buffer)

    The parameters stay the caller's nn.Parameters (updated in place, version counters bumped), so checkpoints, the
    render entry points and scene_io see them as after a torch.optim.Adam step with the same hyper-parameters.
    grad_mode=MLP_TC_HALF runs the backward's dgrad / wgrad GEMMs on tensor cores (see render_backward);
    grad_mode=GRAD_TC_FULL (step_rays only) also its forward recompute (see render_backward_rays).  Under
    torch.use_deterministic_algorithms(True) every step is bit-reproducible: two runs from the same start on the same
    batches end with identical parameters, volume and losses (see render_backward).  `step` takes marched samples;
    `step_rays` takes the rays and marches them inside the backward kernel (three launches)."""

    def __init__(self, network_fn, volume, imgs, pose_ref, lr=5e-4, betas=(0.9, 0.999), eps=1e-8, white_bkgd=False,
                 grad_mode=_lib.MLP_FP32):
        _check_grad_mode(grad_mode, rays=True)
        self.grad_mode = grad_mode
        self.network_fn, self.volume, self.imgs, self.pose_ref = network_fn, volume, imgs, pose_ref
        self.lr, self.betas, self.eps, self.white_bkgd = float(lr), (float(betas[0]), float(betas[1])), float(eps), bool(white_bkgd)
        self.step_count = 0
        self.params = network_fn.ordered_params()
        dev = self.params[0].device
        self.m = [torch.zeros_like(p) for p in self.params]
        self.v = [torch.zeros_like(p) for p in self.params]
        self.g = [torch.zeros_like(p) for p in self.params]
        fv = volume.feat_volume
        if fv.dim() != 5 or fv.shape[0] != 1 or fv.shape[1] != 8 or not fv.is_cuda or fv.dtype != torch.float32:
            raise RuntimeError("FineTuner: volume.feat_volume must be a CUDA fp32 tensor [1,8,D,H,W]")
        _, _, D, Hp, Wp = fv.shape
        self.nvox = D * Hp * Wp
        cl = fv.detach()[0].permute(1, 2, 3, 0)
        if cl.is_contiguous():
            self.planar = 0                                   # channels-last storage (what MVSNet.forward returns)
        elif fv.is_contiguous():
            self.planar = 1                                   # checkpoint layout [8][nvox]
        else:
            raise RuntimeError("FineTuner: feat_volume must be contiguous either planar or channels-last")
        self.vol_m = torch.zeros_like(fv.detach())
        self.vol_v = torch.zeros_like(fv.detach())
        self.vol_g = torch.zeros(D, Hp, Wp, 8, dtype=torch.float32, device=dev)   # zeroed again by every Adam step
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self._numel = (C.c_int * len(self.params))(*[p.numel() for p in self.params])

    def step(self, rays_pts, rays_ndc, z_vals, rays_dir, target_rgb, lr=None, want_forward=False, t_stop=None):
        """One optimisation step on a batch.  Returns (loss [1] device tensor -- img2mse of this batch BEFORE the
        update, as the reference logs it -- and (rgb, depth) of the forward pass when `want_forward`).  `t_stop`: early
        ray termination, as in render_backward -- the step trains the render truncated where each ray's transmittance
        falls below t_stop, and skips the work of the samples behind."""
        _check_grad_mode(self.grad_mode)
        lr = self.lr if lr is None else float(lr)
        self.step_count += 1
        self.loss.zero_()
        _, _, rgb, depth = render_backward(self.pose_ref, rays_pts, rays_ndc, z_vals, rays_dir, self.volume, self.imgs,
                                           self.network_fn, self.white_bkgd, target_rgb=target_rgb, want_volume_grad=True,
                                           grad_volume=self.vol_g, grad_mlp=self.g, want_forward=want_forward,
                                           loss_out=self.loss, grad_mode=self.grad_mode, t_stop=t_stop)
        self._adam(lr)
        return self.loss, (rgb, depth)

    def step_rays(self, rays, target_rgb, near_far, pad, N_samples=128, lindisp=False, perturb=1.0, generator=None,
                  lr=None, want_forward=False, t_stop=None, density=None, N_importance=0):
        """One optimisation step on a batch of rays [N,8] = (o, d, near, far), as train_mvs_nerf_finetuning_pl.py:140-164
        feeds it: the ray march (ray_marcher with `perturb`) and the NDC conversion run inside the backward kernel
        (render_backward_rays).  With perturb > 0 the jitter is drawn as ray_marcher draws it, `perturb *
        torch.rand((N, N_samples))` (from `generator`, or the default generator), so switching a run from
        `step(*ray_marcher(...))` to step_rays consumes the same random stream.  `near_far` / `pad` as in render_rays.
        `t_stop`: early ray termination, as in render_backward_rays -- the step trains the render truncated where each
        ray's transmittance falls below t_stop, and skips the work of the samples behind.  Returns what `step` returns.

        `density` (a `Density` from build_density, or a CUDA fp32 sigma tensor [D, Hp, Wp]) with `N_importance` = K >= 1:
        the reference's --use_density_volume --N_importance K step (train_mvs_nerf_finetuning_pl.py:150-164).  The
        jitter [N, N_samples] and then u [N, K] are drawn from `generator` in the reference's order (ray_marcher, then
        sample_pdf); mvsn_sample_importance marches the jittered coarse samples, draws K more from the grid and sorts
        them; the step is then `step` on those N_samples + K samples (render_backward).  N_samples + K <= 128 (the
        backward's limit) and grad_mode MLP_FP32 or MLP_TC_HALF: otherwise RuntimeError before any launch."""
        lr = self.lr if lr is None else float(lr)
        if density is not None or N_importance:
            S, K = _importance_shape(N_samples, N_importance, "FineTuner.step_rays", max_total=128)
            if density is None:
                raise RuntimeError("FineTuner.step_rays: N_importance needs density= (a Density from build_density)")
            if self.grad_mode == _lib.GRAD_TC_FULL:
                raise RuntimeError("FineTuner.step_rays: importance sampling trains through the samples entries, which "
                                   "run MLP_FP32 or MLP_TC_HALF (grad_mode GRAD_TC_FULL given)")
            sigma = _density_sigma(density, "FineTuner.step_rays", near_far, pad, lindisp)
            rays = _lib.dev_f32(rays.detach(), "rays")
            n = rays.shape[0]
            jitter = None
            if perturb > 0:
                jitter = perturb * torch.rand((n, S), device=rays.device, generator=generator)
            u = torch.rand((n, K), device=rays.device, generator=generator)
            z, pts, ndc = sample_importance(rays, sigma, self.volume, self.imgs, self.pose_ref, self.network_fn, near_far,
                                            pad, N_samples=S, N_importance=K, lindisp=lindisp, jitter=jitter, u=u)
            return self.step(pts, ndc, z, rays[:, 3:6], target_rgb, lr=lr, want_forward=want_forward, t_stop=t_stop)
        rays = _lib.dev_f32(rays.detach(), "rays")
        jitter = None
        if perturb > 0:
            jitter = perturb * torch.rand((rays.shape[0], int(N_samples)), device=rays.device, generator=generator)
        self.step_count += 1
        self.loss.zero_()
        _, _, rgb, depth = render_backward_rays(rays, self.volume, self.imgs, self.pose_ref, self.network_fn, near_far,
                                                pad, N_samples=N_samples, lindisp=lindisp, jitter=jitter,
                                                white_bkgd=self.white_bkgd, target_rgb=target_rgb, want_volume_grad=True,
                                                grad_volume=self.vol_g, grad_mlp=self.g, want_forward=want_forward,
                                                loss_out=self.loss, grad_mode=self.grad_mode, t_stop=t_stop)
        self._adam(lr)
        return self.loss, (rgb, depth)

    def _adam(self, lr):
        """mvsn_adam_step + mvsn_adam_step_volume on the gradients of the step's backward launch."""
        lib = _lib.load()
        dev = self.params[0].device
        fv = self.volume.feat_volume
        with torch.cuda.device(dev):
            _lib.check(lib.mvsn_adam_step(_lib.ptr_array([p.detach() for p in self.params]), _lib.ptr_array(self.g),
                                          _lib.ptr_array(self.m), _lib.ptr_array(self.v), self._numel, len(self.params),
                                          lr, self.betas[0], self.betas[1], self.eps, self.step_count, _lib.stream_ptr()),
                       "mvsn_adam_step")
            _lib.check(lib.mvsn_adam_step_volume(_lib.ptr(fv.detach()), _lib.ptr(self.vol_g), _lib.ptr(self.vol_m),
                                                 _lib.ptr(self.vol_v), self.nvox, self.planar, lr, self.betas[0],
                                                 self.betas[1], self.eps, self.step_count, _lib.stream_ptr()),
                       "mvsn_adam_step_volume")
        # the parameters changed behind PyTorch's back: bump their version counters (weight-image / volume caches)
        torch.autograd.graph.increment_version([p for p in self.params] + [fv])


def ray_marcher(rays, N_samples=64, lindisp=False, perturb=0):
    """data/ray_utils.py:152-197 (without the bbox branch): sample points along rays [N,8] = (o, d, near, far).
    Returns (xyz [N,S,3], rays_o [N,3], rays_d [N,3], z_vals [N,S]).  Host-side mirror for the training callers
    (perturb > 0 draws torch.rand like the reference); inference uses the fused render_rays entry instead."""
    n = rays.shape[0]
    rays_o, rays_d = rays[:, 0:3], rays[:, 3:6]
    near, far = rays[:, 6:7], rays[:, 7:8]
    z_steps = torch.linspace(0, 1, N_samples, device=rays.device)
    if not lindisp:
        z_vals = near * (1 - z_steps) + far * z_steps
    else:
        z_vals = 1 / (1 / near * (1 - z_steps) + 1 / far * z_steps)
    z_vals = z_vals.expand(n, N_samples)
    if perturb > 0:
        mid = 0.5 * (z_vals[:, :-1] + z_vals[:, 1:])
        upper = torch.cat([mid, z_vals[:, -1:]], -1)
        lower = torch.cat([z_vals[:, :1], mid], -1)
        z_vals = lower + (upper - lower) * (perturb * torch.rand(z_vals.shape, device=rays.device))
    xyz = rays_o.unsqueeze(1) + rays_d.unsqueeze(1) * z_vals.unsqueeze(2)
    return xyz, rays_o, rays_d, z_vals


def _matmul3(p, m):
    """p [M,3] @ m[3,3]^T as an FMA-capable BLAS computes it for fp32: row r = fma(p2, m[r,2], fma(p1, m[r,1], p0 m[r,0])),
    each fma formed in fp64 (where the product of two floats is exact) and rounded to fp32.  torch.matmul's rounding of
    these 3-term dot products depends on the CPU's BLAS code path (without FMA it rounds every product); this order is
    the one of the reference run on AVX2 / AVX-512 hosts and of the kernels' ndc_of_point, on any host.  Other dtypes:
    torch.matmul."""
    if p.dtype != torch.float32 or m.dtype != torch.float32:
        return torch.matmul(p, m.t())
    pd, md = p.double(), m.double()
    out = p[:, :1] * m[:, 0].reshape(1, 3)
    for k in (1, 2):
        out = (pd[:, k:k + 1] * md[:, k].reshape(1, 3) + out.double()).float()
    return out


def get_ndc_coordinate(w2c_ref, intrinsic_ref, point_samples, inv_scale, near=2, far=6, pad=0, lindisp=False):
    """utils.py:112-146 (projection branch): world points [N,S,3] -> volume coordinates in [0,1].  The two 3x3 products
    are rounded as _matmul3 states, the same on every host."""
    n, s = point_samples.shape[:2]
    p = point_samples.reshape(-1, 3)
    p = _matmul3(p, w2c_ref[:3, :3]) + w2c_ref[:3, 3:].reshape(1, 3)
    q = _matmul3(p, intrinsic_ref)
    q[:, :2] = (q[:, :2] / q[:, -1:] + 0.0) / inv_scale.reshape(1, 2)
    if not lindisp:
        q[:, 2] = (q[:, 2] - near) / (far - near)
    else:
        q[:, 2] = (1.0 / q[:, 2] - 1.0 / near) / (1.0 / far - 1.0 / near)
    if pad > 0:
        w_feat, h_feat = (inv_scale + 1) / 4.0
        q[:, 1] = q[:, 1] * h_feat / (h_feat + pad * 2) + pad / (h_feat + pad * 2)
        q[:, 0] = q[:, 0] * w_feat / (w_feat + pad * 2) + pad / (w_feat + pad * 2)
    return q.view(n, s, 3)


def finetune_step_timing(dev, weights_npz, steps=20, warmup=5, batch=1024, n_samples=128, grad_mode=_lib.MLP_FP32):
    """bench.py's BASELINE-config-3 entry: fine-tuning steps on a Blender-shaped scene (800x800, pad 0, white_bkgd,
    near_far [2, 6]; encoding volume 8x128x200x200), 1024 rays x 128 samples per step, perturb = 1 -- the fused
    FineTuner step and, beside it, the same step through `rendering` under autograd + torch.optim.Adam.  `grad_mode`
    selects the arithmetic of the backward's GEMMs in both."""
    from . import synthetic
    fn, mvs = MVSNeRF().to(dev), MVSNet().to(dev).train()
    load_weights_npz(fn, mvs, weights_npz)
    sc = synthetic.make_scene(800, 800, pad=0, seed=3, near_far=(2.0, 6.0))
    d = sc.to(dev)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=0)
    rays_all = synthetic.scene_rays(sc).to(dev)
    target_all = d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
    inv_scale = torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)

    def batch_of():
        idx = torch.randint(0, rays_all.shape[0], (batch,), device=dev, generator=gen)
        rays, tgt = rays_all[idx], target_all[idx]
        xyz, _, rays_d, z = ray_marcher(rays, N_samples=n_samples, perturb=1.0)
        ndc = get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz, inv_scale,
                                 near=sc.near_far[0], far=sc.near_far[1], pad=0)
        return xyz, ndc, z, rays_d, tgt

    def timed(fn_step):
        for _ in range(warmup):
            fn_step(*batch_of())
        torch.cuda.synchronize()
        ts = []
        for _ in range(steps):
            b = batch_of()
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn_step(*b); e.record(); e.synchronize()
            ts.append(a.elapsed_time(e))
        ts.sort()
        return ts[len(ts) // 2]

    out = {"rays": batch, "n_samples": n_samples, "volume": list(vol.shape), "white_bkgd": True}
    volume = RefVolume(vol.detach().clone()).to(dev)
    tuner = FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=5e-4, white_bkgd=True, grad_mode=grad_mode)
    losses = []
    out["fused_ms"] = timed(lambda xyz, ndc, z, rd, tgt: losses.append(tuner.step(xyz, ndc, z, rd, tgt)[0].clone()))
    out["fused_loss_first_last"] = [float(losses[0]), float(losses[-1])]
    # the reference's own step shape: rendering under autograd (kernel forward + kernel backward) + torch.optim.Adam
    fn2 = MVSNeRF().to(dev)
    load_weights_npz(fn2, None, weights_npz)
    volume2 = RefVolume(vol.detach().clone()).to(dev)
    opt = torch.optim.Adam(list(fn2.parameters()) + list(volume2.parameters()), lr=5e-4, betas=(0.9, 0.999))
    from types import SimpleNamespace
    args = SimpleNamespace(use_color_volume=False)

    def autograd_step(xyz, ndc, z, rd, tgt):
        rgb = rendering(args, d.pose_source, xyz, ndc, z, None, rd, volume2, d.imgs_raw, network_fn=fn2, white_bkgd=True,
                        want_aux=True, grad_mode=grad_mode)[0]
        loss = torch.mean((rgb - tgt) ** 2)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    out["autograd_adam_ms"] = timed(autograd_step)
    out["note"] = ("median CUDA-event ms per step incl. ray marching (torch ops) ; fused = FineTuner.step (mvsn_render_backward "
                   "+ mvsn_adam_step + mvsn_adam_step_volume); autograd = backend.rendering under autograd (kernel backward) "
                   "+ torch.optim.Adam; README.md's reference figure is ~15 min for 10k such steps")
    return out


def _ordered_named_params(network_fn):
    """(name, parameter) in MVSNeRF.ordered_params() order."""
    by_id = {id(p): n for n, p in network_fn.named_parameters()}
    return [(by_id[id(p)], p) for p in network_fn.ordered_params()]


_tsteps = {}
_occ_workspace = {}          # per device: the range table of render_rays(occupancy=), grown to the largest batch


class Occupancy:
    """An occupancy grid of a scene's density for empty-space skipping (`render_rays(..., occupancy=)`): one bit per cell
    of the encoding volume's D x Hp x Wp node grid in NDC (`bits`, int32 words, see mvsn_build_occupancy), and the
    geometry it was built for -- the rays' NDC mapping must be the same (near_far, pad, lindisp) for it to apply."""

    def __init__(self, bits, D, Hp, Wp, near_far, pad, lindisp, dilate):
        self.bits, self.D, self.Hp, self.Wp = bits, int(D), int(Hp), int(Wp)
        self.near_far, self.pad, self.lindisp, self.dilate = (float(near_far[0]), float(near_far[1])), float(pad), \
            bool(lindisp), int(dilate)

    def cells(self):
        """bool [D, Hp, Wp]: cell (d, y, x) occupied (the last slab of each axis is always False)."""
        n = self.D * self.Hp * self.Wp
        shifts = torch.arange(32, dtype=torch.int32, device=self.bits.device)
        return ((self.bits.view(-1, 1) >> shifts) & 1).bool().reshape(-1)[:n].view(self.D, self.Hp, self.Wp)

    def fraction(self):
        """occupied cells / all (D - 1) (Hp - 1) (Wp - 1) cells"""
        return float(self.cells().sum()) / ((self.D - 1) * (self.Hp - 1) * (self.Wp - 1))

    def _grid(self):
        return _lib.OccupancyGrid(self.bits.data_ptr(), self.D, self.Hp, self.Wp)


def build_occupancy(volume_feature, imgs, pose_ref, network_fn, near_far, pad, lindisp=False, dilate=1):
    """The occupancy grid of a scene for `render_rays(..., occupancy=)` (mvsn_build_occupancy): sigma at every node of the
    volume's grid (the split tensor-core MLP, the node as the sample's NDC, the world point from inverting
    get_ndc_coordinate with `near_far` / `pad` / `lindisp`), a cell occupied when alpha > 0 at any of its eight corners,
    then dilated by `dilate` cells (0..8).  fp32 and fp16 volumes.  Returns an `Occupancy`.

    The grid depends on the volume, the MLP, the source images and cameras: it is cached on their version counters (a
    repeated call returns the same object), so call build_occupancy again after fine-tuning -- an `Occupancy` held from
    before describes the old scene."""
    dilate = int(dilate)
    if not 0 <= dilate <= 8:
        raise RuntimeError(f"build_occupancy: dilate={dilate} must be in 0..8")
    owner = volume_feature.feat_volume if isinstance(volume_feature, nn.Module) else volume_feature
    if not owner.is_cuda:
        raise RuntimeError("build_occupancy: the encoding volume must be a CUDA tensor; mvsnerf_b200 has no CPU path")
    params = network_fn.ordered_params()
    tensors = [owner, imgs, pose_ref["w2cs"], pose_ref["intrinsics"]] + list(params)
    args = (float(near_far[0]), float(near_far[1]), float(pad), bool(lindisp), dilate)
    hit = _cache.get("occupancy")
    if hit is not None and hit[1] == args and len(hit[0]) == len(tensors) and \
            all(r() is t and v == t._version for (r, v), t in zip(hit[0], tensors)):
        cache_stats["hit"] += 1
        return hit[2]
    cache_stats["miss"] += 1
    lib = _lib.load()
    sc, keep = _make_scene(pose_ref, volume_feature, imgs, network_fn, False, _lib.MLP_TC_SPLIT, half_ok=True)
    dev = owner.device
    rp = _lib.RayParams(args[0], args[1], args[2], int(args[3]))
    bits = torch.empty(lib.mvsn_occupancy_bytes(sc.D, sc.Hp, sc.Wp) // 4, dtype=torch.int32, device=dev)
    need = lib.mvsn_build_occupancy_workspace_bytes(sc.D, sc.Hp, sc.Wp)
    if need == 0:
        raise RuntimeError(f"build_occupancy: volume {sc.D}x{sc.Hp}x{sc.Wp} (every dim >= 2)")
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.mvsn_build_occupancy(C.byref(sc), C.byref(rp), dilate, _lib.ptr(bits), _lib.ptr(ws), need,
                                            _lib.stream_ptr()), "mvsn_build_occupancy")
    del keep
    occ = Occupancy(bits, sc.D, sc.Hp, sc.Wp, near_far, pad, lindisp, dilate)
    _cache["occupancy"] = ([(weakref.ref(t), t._version) for t in tensors], args, occ)
    return occ


# --------------------------------------------------------------------------------------------
# importance sampling from a density grid (data/ray_utils.py:98-141 sample_pdf, :199-224 ray_marcher_fine)
# --------------------------------------------------------------------------------------------
IMPORTANCE_CHUNK_RAYS = 32768   # rays per sampler + render launch pair in render_rays (a multiple of 32)
_imp_buffers = {}               # per device: z / pts / ndc / dirs of one chunk, grown to the largest


class Density:
    """A density grid of a scene for importance sampling: sigma [D, Hp, Wp] (fp32, the reference's density_volume
    layout) at the encoding volume's nodes in NDC, and the geometry it was built for -- the rays' NDC mapping must be
    the same (near_far, pad, lindisp) for it to apply."""

    def __init__(self, sigma, near_far, pad, lindisp):
        self.sigma = sigma
        self.D, self.Hp, self.Wp = (int(v) for v in sigma.shape)
        self.near_far, self.pad, self.lindisp = (float(near_far[0]), float(near_far[1])), float(pad), bool(lindisp)


def build_density(volume_feature, imgs, pose_ref, network_fn, near_far, pad, lindisp=False):
    """The density grid of a scene (mvsn_build_density): sigma = relu(alpha_linear(h)) at every node of the volume's
    grid, the node as the sample's NDC and the world point from inverting get_ndc_coordinate with `near_far` / `pad` /
    `lindisp` (the nodes of build_occupancy), evaluated in fp32 by the FFMA tile.  fp32 and fp16 volumes (an fp16
    volume gives the grid of its fp32 upcast, bit for bit).  Returns a `Density`.

    This is the reference's update_density_volume (train_mvs_nerf_finetuning_pl.py:91-99) with sigma taken where the
    renderer evaluates it: at the node's NDC, not at its positionally encoded world point (DESIGN §5).  The grid is
    cached on the version counters of the volume, the MLP, the images and cameras, as build_occupancy's: FineTuner's
    Adam step bumps them, so calling build_density every 200 steps rebuilds it after an update."""
    owner = volume_feature.feat_volume if isinstance(volume_feature, nn.Module) else volume_feature
    if not owner.is_cuda:
        raise RuntimeError("build_density: the encoding volume must be a CUDA tensor; mvsnerf_b200 has no CPU path")
    params = network_fn.ordered_params()
    tensors = [owner, imgs, pose_ref["w2cs"], pose_ref["intrinsics"]] + list(params)
    args = (float(near_far[0]), float(near_far[1]), float(pad), bool(lindisp))
    hit = _cache.get("density")
    if hit is not None and hit[1] == args and len(hit[0]) == len(tensors) and \
            all(r() is t and v == t._version for (r, v), t in zip(hit[0], tensors)):
        cache_stats["hit"] += 1
        return hit[2]
    cache_stats["miss"] += 1
    lib = _lib.load()
    sc, keep = _make_scene(pose_ref, volume_feature, imgs, network_fn, False, _lib.MLP_FP32, half_ok=True, half_fp32=True)
    dev = owner.device
    rp = _lib.RayParams(args[0], args[1], args[2], int(args[3]))
    need = lib.mvsn_build_density_workspace_bytes(sc.D, sc.Hp, sc.Wp)
    if need == 0:
        raise RuntimeError(f"build_density: volume {sc.D}x{sc.Hp}x{sc.Wp} (every dim >= 2)")
    sigma = torch.empty(sc.D, sc.Hp, sc.Wp, dtype=torch.float32, device=dev)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.mvsn_build_density(C.byref(sc), C.byref(rp), _lib.ptr(sigma), _lib.ptr(ws), need,
                                          _lib.stream_ptr()), "mvsn_build_density")
    del keep
    den = Density(sigma, near_far, pad, lindisp)
    _cache["density"] = ([(weakref.ref(t), t._version) for t in tensors], args, den)
    return den


def _importance_shape(N_samples, N_importance, who, max_total=1024):
    """(S, K) after the sampler's limits: 3 <= S, 1 <= K, S + K <= max_total"""
    S, K = int(N_samples), int(N_importance)
    if S < 3 or K < 1:
        raise RuntimeError(f"{who}: N_samples={S}, N_importance={K} (importance sampling needs N_samples >= 3 and "
                           "N_importance >= 1)")
    if S + K > max_total:
        raise RuntimeError(f"{who}: N_samples + N_importance = {S + K} exceeds {max_total}"
                           + (" (the fine-tuning backward's N_samples limit)" if max_total == 128 else ""))
    return S, K


def _density_sigma(density, who, near_far=None, pad=None, lindisp=None):
    """The sigma tensor of a `Density` (checked against the rays' geometry when it is given) or of a CUDA fp32 [D,H,W]
    tensor (the reference's density_volume)."""
    if isinstance(density, Density):
        if near_far is not None and (density.near_far != (float(near_far[0]), float(near_far[1])) or
                                     density.pad != float(pad) or density.lindisp != bool(lindisp)):
            raise RuntimeError(f"{who}: the density grid was built for another near_far / pad / lindisp")
        return density.sigma
    if isinstance(density, torch.Tensor) and density.is_cuda and density.dtype == torch.float32 and density.dim() == 3:
        return density.detach().contiguous()
    raise RuntimeError(f"{who}: density must be a Density from build_density or a CUDA fp32 tensor [D, H, W]")


def _sample_importance_launch(sc, rp, sigma, rays, t_steps, jitter, z_vals, ndc_in, u, N, S, K, z, pts, ndc):
    grid = _lib.DensityGrid(sigma.data_ptr(), *[int(v) for v in sigma.shape])
    _lib.check(_lib.load().mvsn_sample_importance(
        None if sc is None else C.byref(sc), None if rp is None else C.byref(rp), C.byref(grid), _lib.ptr(rays),
        _lib.ptr(t_steps), _lib.ptr(jitter), _lib.ptr(z_vals), _lib.ptr(ndc_in), _lib.ptr(u), int(N), int(S), int(K),
        _lib.ptr(z), _lib.ptr(pts), _lib.ptr(ndc), _lib.stream_ptr()), "mvsn_sample_importance")


def _opt_draws(t, n, k, name, who):
    if t is None:
        return None
    t = _lib.dev_f32(t.detach(), name)
    if tuple(t.shape) != (n, k):
        raise RuntimeError(f"{who}: {name} must be [{n}, {k}], got {tuple(t.shape)}")
    return t


def sample_importance(rays, density, volume_feature, imgs, pose_ref, network_fn, near_far, pad, N_samples=64,
                      N_importance=64, lindisp=False, jitter=None, u=None):
    """The importance sampler on rays [N,8] (mvsn_sample_importance, marched source): ray_marcher with `N_samples`,
    `lindisp` and the stratification `jitter` [N, N_samples] (= perturb * u as ray_marcher draws it; None: none),
    then ray_marcher_fine's K = `N_importance` samples from `density` with the uniform draws `u` [N, K] (None:
    torch.linspace(0, 1, K)).  Returns (z [N,S+K] sorted, pts [N,S+K,3] = o + d z, ndc [N,S+K,3]): the samples
    `rendering` / `FineTuner.step` take, the NDC by the render's get_ndc_coordinate for `near_far` / `pad`."""
    S, K = _importance_shape(N_samples, N_importance, "sample_importance")
    sigma = _density_sigma(density, "sample_importance", near_far, pad, lindisp)
    rays = _lib.dev_f32(rays.detach(), "rays")
    n, dev = rays.shape[0], rays.device
    jitter = _opt_draws(jitter, n, S, "jitter", "sample_importance")
    u = _opt_draws(u, n, K, "u", "sample_importance")
    sc, keep = _make_scene(pose_ref, volume_feature, imgs, network_fn, False, _lib.MLP_FP32)
    rp = _lib.RayParams(float(near_far[0]), float(near_far[1]), float(pad), int(bool(lindisp)))
    z = torch.empty(n, S + K, dtype=torch.float32, device=dev)
    pts = torch.empty(n, S + K, 3, dtype=torch.float32, device=dev)
    ndc = torch.empty(n, S + K, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _sample_importance_launch(sc, rp, sigma, rays, _tsteps_of(S, dev), jitter, None, None, u, n, S, K, z, pts, ndc)
    del keep
    return z, pts, ndc


def ray_marcher_fine(rays, density_volume, z_vals, pts_NDC, N_importance=64, lindisp=False):
    """data/ray_utils.py:199-224 on the GPU (mvsn_sample_importance, the caller's coarse samples): K = N_importance
    depths per ray drawn by inverse-CDF sampling of the density grid's weights along z_vals [N,S] (looked up at
    pts_NDC [N,S,3]), merged with z_vals and sorted.  Returns (xyz [N,S+K,3], rays_o, rays_d, z_vals [N,S+K]), as the
    reference does; the caller recomputes the NDC.  `density_volume`: a `Density` or a CUDA fp32 tensor [D,H,W].  u is
    drawn as sample_pdf draws it, torch.rand((N, K)) from the default generator on the rays' device, so a seeded run
    consumes the same stream.  The grid is looked up at pts_NDC itself, the volume's own mapping, where the reference
    maps the coordinate twice (DESIGN §5).  `lindisp` is accepted and unused, as in the reference."""
    n, S = int(z_vals.shape[0]), int(z_vals.shape[1])
    S, K = _importance_shape(S, N_importance, "ray_marcher_fine")
    sigma = _density_sigma(density_volume, "ray_marcher_fine")
    r = _lib.dev_f32(rays.detach(), "rays")
    z_in = _lib.dev_f32(z_vals.detach(), "z_vals")
    ndc_in = _lib.dev_f32(pts_NDC.detach(), "pts_NDC")
    if tuple(ndc_in.shape) != (n, S, 3) or r.shape[0] != n:
        raise RuntimeError(f"ray_marcher_fine: rays [{n},8], z_vals [{n},{S}] and pts_NDC [{n},{S},3] expected, got "
                           f"{tuple(r.shape)}, {tuple(z_vals.shape)} and {tuple(pts_NDC.shape)}")
    dev = r.device
    u = torch.rand((n, K), device=rays.device)
    z = torch.empty(n, S + K, dtype=torch.float32, device=dev)
    xyz = torch.empty(n, S + K, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _sample_importance_launch(None, None, sigma, r, None, None, z_in, ndc_in, u, n, S, K, z, xyz, None)
    return xyz, rays[:, 0:3], rays[:, 3:6], z


def render_density(network_fn, rays_pts, density_feature, network_query_fn, chunk=1024 * 5):
    """renderer.render_density (renderer.py:167-177), unchanged: network_query_fn(pts, None, feats, network_fn) over
    chunks of `chunk` points, concatenated -- what an unchanged update_density_volume calls.  build_density computes the
    grid in one launch instead."""
    densities = []
    device = density_feature.device
    for i in range(0, rays_pts.shape[0], chunk):
        densities.append(network_query_fn(rays_pts[i:i + chunk].to(device), None, density_feature[i:i + chunk],
                                          network_fn))
    return torch.cat(densities)


def _render_rays_importance(rays, volume_feature, imgs, pose_ref, network_fn, near_far, pad, N_samples, white_bkgd,
                            lindisp, mode, out, t_stop, tiles_done, density, N_importance, importance_u):
    """render_rays(density=, N_importance=): per chunk of IMPORTANCE_CHUNK_RAYS rays, mvsn_sample_importance (linspace
    coarse samples, their NDC) then mvsn_render_samples[_stop] on the S + K samples."""
    if density is None:
        raise RuntimeError("render_rays: N_importance needs density= (a Density from build_density)")
    S, K = _importance_shape(N_samples, N_importance, "render_rays")
    sigma = _density_sigma(density, "render_rays", near_far, pad, lindisp)
    if t_stop is not None:
        t_stop = float(t_stop)
        if not t_stop >= 0.0:
            raise RuntimeError(f"render_rays: t_stop={t_stop} must be >= 0")
        _check_counter(tiles_done, "render_rays", "tiles_done", torch.int64, 1, rays.device)
    lib = _lib.load()
    rays = _lib.dev_f32(rays, "rays")
    N, dev, M = rays.shape[0], rays.device, S + K
    u = _opt_draws(importance_u, N, K, "importance_u", "render_rays")
    sc, keep = _make_scene(pose_ref, volume_feature, imgs, network_fn, white_bkgd, mode, half_ok=True)
    rp = _lib.RayParams(float(near_far[0]), float(near_far[1]), float(pad), int(bool(lindisp)))
    if out is not None:
        rgb, depth = out
    else:
        rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
    chunk = max(1, min(N, IMPORTANCE_CHUNK_RAYS))
    buf = _imp_buffers.get(dev)
    if buf is None or buf.numel() < chunk * M * 7 + chunk * 3:
        buf = torch.empty(chunk * M * 7 + chunk * 3, dtype=torch.float32, device=dev)
        _imp_buffers[dev] = buf
    t_steps = _tsteps_of(S, dev)
    with torch.cuda.device(dev):
        for c0 in range(0, N, chunk):
            n = min(chunk, N - c0)
            r = rays[c0:c0 + n]
            z, pts, ndc = buf[:n * M], buf[n * M:4 * n * M], buf[4 * n * M:7 * n * M]
            dirs = buf[7 * n * M:7 * n * M + 3 * n].view(n, 3)
            dirs.copy_(r[:, 3:6])
            _sample_importance_launch(sc, rp, sigma, r, t_steps, None, None, None, None if u is None else u[c0:c0 + n],
                                      n, S, K, z, pts, ndc)
            if t_stop is None:
                _lib.check(lib.mvsn_render_samples(C.byref(sc), _lib.ptr(pts), _lib.ptr(ndc), _lib.ptr(z), _lib.ptr(dirs),
                                                   n, M, _lib.ptr(rgb[c0:c0 + n]), _lib.ptr(depth[c0:c0 + n]), None,
                                                   None, None, _lib.stream_ptr()), "mvsn_render_samples")
            else:
                _lib.check(lib.mvsn_render_samples_stop(C.byref(sc), _lib.ptr(pts), _lib.ptr(ndc), _lib.ptr(z),
                                                        _lib.ptr(dirs), n, M, t_stop, _lib.ptr(rgb[c0:c0 + n]),
                                                        _lib.ptr(depth[c0:c0 + n]), _lib.ptr(tiles_done),
                                                        _lib.stream_ptr()), "mvsn_render_samples_stop")
    del keep
    return rgb, depth


def render_rays(rays, volume_feature, imgs, pose_ref, network_fn, near_far, pad, N_samples=128,
                white_bkgd=False, lindisp=False, mlp_mode=None, out=None, sink=None, t_stop=None, tiles_done=None,
                occupancy=None, density=None, N_importance=0, importance_u=None):
    """Fused-caller entry: one launch renders all `rays` [N,8] = (o, d, near, far).

    Replaces the notebooks' per-chunk loop `ray_marcher -> get_ndc_coordinate -> rendering`
    (renderer_video.ipynb "DTU video rendering"; data/ray_utils.py:152-197, utils.py:112-146) with
    perturb = 0.  `near_far` / `pad` are the arguments the reference passes to get_ndc_coordinate
    (near_far of the source views, pad * imgScale_test).  Returns (rgb [N,3], depth [N]).

    `sink` (a lib.PeerSink from distributed.PeerFrame.sink): the kernel epilogue additionally stores every pixel
    as (r, g, b, depth) into all ranks' copies of the assembled frame (mvsn_render_rays_to_peers); with a sink and
    no `out`, nothing else is written and (None, None) is returned.

    `t_stop` (a float >= 0, tensor-core modes): early ray termination (mvsn_render_rays_stop) -- a group of up to 32
    neighbouring rays stops two tiles (four samples at frame sizes) after every ray in it has transmittance < t_stop, so
    each channel differs from the full render by less than t_stop (t_stop = 0: bit-identical).  `tiles_done`: an
    optional CUDA int64 tensor [1] the number of computed 64-sample tiles is added to.  Not combinable with `sink`.

    `occupancy` (an `Occupancy` from build_occupancy for this scene, near_far, pad and lindisp; tensor-core modes):
    empty-space skipping (mvsn_render_rays_occ) -- each group of rays computes only the tiles from its first to its last
    sample in an occupied cell, and a group with none stores rgb 0 (1 with white_bkgd) and depth 0.  A pixel is
    bit-identical to the full render whenever the full render's alpha is exactly 0 on every skipped sample; the grid is a
    heuristic (DESIGN §4 K-C).  Composes with `t_stop` (without it the call runs with t_stop = 0, which never stops);
    `tiles_done` works with either.  Not combinable with `sink`.

    A float16 `volume_feature` is read as fp16 in the tensor-core modes (half the resident bytes): the result is
    bit-identical to rendering `volume.float()`.  Channels-last storage (MVSNet.forward(..., volume_dtype=torch.float16),
    or `.half()` of an fp32 MVSNet volume) is read in place; other layouts are converted once per tensor version.

    `density` (a `Density` from build_density for this near_far / pad / lindisp, or a CUDA fp32 sigma tensor
    [D, Hp, Wp]) with `N_importance` = K >= 1: importance sampling (the reference's --use_density_volume --N_importance).
    Each ray's N_samples linspace samples and K more drawn from the grid by inverse-CDF sampling (mvsn_sample_importance),
    sorted, are rendered by the samples entry (mvsn_render_samples, or mvsn_render_samples_stop with t_stop) in any
    mlp_mode, in chunks of IMPORTANCE_CHUNK_RAYS rays.  `importance_u` [N, K]: the uniform draws (the reference's
    validation draws torch.rand); None draws torch.linspace(0, 1, K) for every ray, a reproducible frame.  Not
    combinable with `occupancy` or `sink`."""
    lib = _lib.load()
    mode = DEFAULT_MLP_MODE if mlp_mode is None else mlp_mode
    if density is not None or N_importance or importance_u is not None:
        if occupancy is not None or sink is not None:
            raise RuntimeError("render_rays: density (importance sampling) cannot be combined with occupancy or sink")
        if t_stop is not None and mode == _lib.MLP_FP32:
            raise RuntimeError("render_rays: t_stop needs a tensor-core mlp_mode (MLP_TC_HALF / TC_PAIR / TC_SPLIT)")
        if t_stop is None and tiles_done is not None:
            raise RuntimeError("render_rays: tiles_done needs t_stop")
        return _render_rays_importance(rays, volume_feature, imgs, pose_ref, network_fn, near_far, pad, N_samples,
                                       white_bkgd, lindisp, mode, out, t_stop, tiles_done, density, N_importance,
                                       importance_u)
    if occupancy is not None:
        if sink is not None:
            raise RuntimeError("render_rays: occupancy cannot be combined with sink (peer frame assembly)")
        if mode == _lib.MLP_FP32:
            raise RuntimeError("render_rays: occupancy needs a tensor-core mlp_mode (MLP_TC_HALF / TC_PAIR / TC_SPLIT)")
        if not isinstance(occupancy, Occupancy):
            raise RuntimeError("render_rays: occupancy must be an Occupancy from build_occupancy")
        if occupancy.near_far != (float(near_far[0]), float(near_far[1])) or occupancy.pad != float(pad) or \
                occupancy.lindisp != bool(lindisp):
            raise RuntimeError("render_rays: the occupancy grid was built for another near_far / pad / lindisp")
        if t_stop is None:
            t_stop = 0.0
    if t_stop is not None:
        t_stop = float(t_stop)
        if sink is not None:
            raise RuntimeError("render_rays: t_stop cannot be combined with sink (peer frame assembly)")
        if mode == _lib.MLP_FP32:
            raise RuntimeError("render_rays: t_stop needs a tensor-core mlp_mode (MLP_TC_HALF / TC_PAIR / TC_SPLIT)")
        if tiles_done is not None and (not tiles_done.is_cuda or tiles_done.device != rays.device
                                       or tiles_done.dtype != torch.int64 or tiles_done.numel() < 1):
            raise RuntimeError(f"render_rays: tiles_done must be a CUDA int64 tensor on the rays' device ({rays.device})")
    elif tiles_done is not None:
        raise RuntimeError("render_rays: tiles_done needs t_stop")
    rays = _lib.dev_f32(rays, "rays")
    N = rays.shape[0]
    dev = rays.device
    S = int(N_samples)
    t_steps = _tsteps_of(S, dev)
    sc, keep = _make_scene(pose_ref, volume_feature, imgs, network_fn, white_bkgd, mode, half_ok=True)
    rp = _lib.RayParams(float(near_far[0]), float(near_far[1]), float(pad), int(bool(lindisp)))
    if out is not None:
        rgb, depth = out
    elif sink is not None:
        rgb = depth = None
    else:
        rgb = torch.empty(N, 3, dtype=torch.float32, device=dev)
        depth = torch.empty(N, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        if occupancy is not None:
            if occupancy.bits.device != dev:
                raise RuntimeError(f"render_rays: the occupancy grid is on {occupancy.bits.device}, the rays on {dev}")
            need = lib.mvsn_render_rays_occ_workspace_bytes(N, S)
            ws = _occ_workspace.get(dev)
            if ws is None or ws.numel() < need:
                ws = torch.empty(need, dtype=torch.uint8, device=dev)
                _occ_workspace[dev] = ws
            grid = occupancy._grid()
            _lib.check(lib.mvsn_render_rays_occ(C.byref(sc), C.byref(rp), _lib.ptr(rays), _lib.ptr(t_steps), N, S, t_stop,
                                                C.byref(grid), _lib.ptr(rgb), _lib.ptr(depth), _lib.ptr(tiles_done),
                                                _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                       "mvsn_render_rays_occ")
        elif t_stop is not None:
            _lib.check(lib.mvsn_render_rays_stop(C.byref(sc), C.byref(rp), _lib.ptr(rays), _lib.ptr(t_steps), N, S,
                                                 t_stop, _lib.ptr(rgb), _lib.ptr(depth), _lib.ptr(tiles_done),
                                                 _lib.stream_ptr()),
                       "mvsn_render_rays_stop")
        elif sink is not None:
            _lib.check(lib.mvsn_render_rays_to_peers(C.byref(sc), C.byref(rp), _lib.ptr(rays), _lib.ptr(t_steps), N, S,
                                                     C.byref(sink), _lib.ptr(rgb), _lib.ptr(depth), _lib.stream_ptr()),
                       "mvsn_render_rays_to_peers")
        else:
            _lib.check(lib.mvsn_render_rays(C.byref(sc), C.byref(rp), _lib.ptr(rays), _lib.ptr(t_steps), N, S,
                                            _lib.ptr(rgb), _lib.ptr(depth), None, None, None, _lib.stream_ptr()),
                       "mvsn_render_rays")
    del keep
    return rgb, depth


def get_rays(directions, c2w, near, far, out=None):
    """data/ray_utils.py:32-53 (get_rays) + the notebooks' `cat([rays_o, rays_d, near, far])` in one launch:
    directions [H,W,3] or [n,3] (camera frame, on the device), c2w [3,4] / [4,4] on the device -> rays [n,8]."""
    lib = _lib.load()
    d = _lib.dev_f32(directions.reshape(-1, 3), "directions")
    m = _lib.dev_f32(c2w, "c2w")
    if m.dim() != 2 or m.shape[1] != 4 or m.shape[0] < 3 or m.device != d.device:
        raise RuntimeError(f"get_rays: c2w must be [3,4] or [4,4] on {d.device}, got {tuple(m.shape)} on {m.device}")
    n = d.shape[0]
    rays = torch.empty(n, 8, dtype=torch.float32, device=d.device) if out is None else out
    with torch.cuda.device(d.device):
        _lib.check(lib.mvsn_make_rays(_lib.ptr(d), _lib.ptr(m), float(near), float(far), n, _lib.ptr(rays), _lib.stream_ptr()),
                   "mvsn_make_rays")
    return rays


class HostFrameRenderer:
    """Host-buffer entry: rays arrive in (pinned) host memory, pixels are returned in host memory.

    This is the call the notebooks' frame loop makes in effect (`rgb.cpu()` / `depth_pred.cpu()` per
    chunk, renderer_video.ipynb DTU cell) collapsed to one H2D copy, one launch, one D2H copy."""

    def __init__(self, n_rays, device):
        self.n, self.device = int(n_rays), torch.device(device)
        self.rays_dev = torch.empty(self.n, 8, dtype=torch.float32, device=self.device)
        self.rgb_dev = torch.empty(self.n, 3, dtype=torch.float32, device=self.device)
        self.depth_dev = torch.empty(self.n, dtype=torch.float32, device=self.device)
        self.rgb_host = torch.empty(self.n, 3, dtype=torch.float32).pin_memory()
        self.depth_host = torch.empty(self.n, dtype=torch.float32).pin_memory()
        self.h2d_bytes = self.n * 8 * 4
        self.d2h_bytes = self.n * 4 * 4

    def render(self, rays_host, volume_feature, imgs, pose_ref, network_fn, near_far, pad, after_launch=None, **kw):
        """`after_launch`: optional callable enqueued between the launch and the read-back (multi-GPU frame assembly:
        distributed.PeerFrame.complete, or an all-gather); `sink=` is forwarded to render_rays."""
        if rays_host.is_cuda or tuple(rays_host.shape) != (self.n, 8):
            raise RuntimeError(f"HostFrameRenderer: expected a host tensor [{self.n}, 8]")
        self.rays_dev.copy_(rays_host, non_blocking=True)
        render_rays(self.rays_dev, volume_feature, imgs, pose_ref, network_fn, near_far, pad,
                    out=(self.rgb_dev, self.depth_dev), **kw)
        if after_launch is not None:
            after_launch()
        self.rgb_host.copy_(self.rgb_dev, non_blocking=True)
        self.depth_host.copy_(self.depth_dev, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return self.rgb_host, self.depth_host

    def render_camera(self, c2w_host, directions_dev, volume_feature, imgs, pose_ref, network_fn, near_far, pad,
                      ray_near_far=None, after_launch=None, **kw):
        """The notebooks' frame loop as it is actually fed (renderer_video.ipynb: one `c2w` per frame, `get_rays` on the
        device): the host input of a frame is the camera pose (pinned [4,4] or [3,4] tensor, 48-64 bytes H2D), the rays
        are generated on the device (mvsn_make_rays) from the resident `directions_dev` [H*W,3], pixels come back to
        pinned host memory."""
        if c2w_host.is_cuda or directions_dev.reshape(-1, 3).shape[0] != self.n:
            raise RuntimeError(f"HostFrameRenderer.render_camera: expected a host c2w and {self.n} device directions")
        if not hasattr(self, "c2w_dev"):
            self.c2w_dev = torch.empty(4, 4, dtype=torch.float32, device=self.device)
        rows = c2w_host.shape[0]
        self.c2w_dev[:rows].copy_(c2w_host, non_blocking=True)
        nf = near_far if ray_near_far is None else ray_near_far
        get_rays(directions_dev, self.c2w_dev, nf[0], nf[1], out=self.rays_dev)
        render_rays(self.rays_dev, volume_feature, imgs, pose_ref, network_fn, near_far, pad,
                    out=(self.rgb_dev, self.depth_dev), **kw)
        if after_launch is not None:
            after_launch()
        self.rgb_host.copy_(self.rgb_dev, non_blocking=True)
        self.depth_host.copy_(self.depth_dev, non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        return self.rgb_host, self.depth_host


# --------------------------------------------------------------------------------------------
# factory (models.py:569-654)
# --------------------------------------------------------------------------------------------
def _embed(x, n_freqs=10):
    """models.py:47-51 (used only by the PyTorch query function below)."""
    freqs = 2.0 ** torch.arange(n_freqs, dtype=x.dtype, device=x.device)
    s = (x.unsqueeze(-2) * freqs.view(-1, 1)).reshape(*x.shape[:-1], -1)
    return torch.cat([x, torch.sin(s), torch.cos(s)], -1)


def _network_query(pts, viewdirs, rays_feats, network_fn, netchunk=1024):
    """run_network_mvs (renderer.py:42-63) for the callers outside `rendering` (alpha-only queries)."""
    x = _embed(pts)
    if rays_feats is not None:
        x = torch.cat([x, rays_feats], -1)
    if viewdirs is not None:
        if viewdirs.dim() != 3:
            viewdirs = viewdirs[:, None].expand(-1, x.shape[1], -1)
        x = torch.cat([x, viewdirs], -1)
    fn = network_fn.forward_alpha if viewdirs is None else network_fn
    return torch.cat([fn(x[i:i + netchunk]) for i in range(0, x.shape[0], netchunk)], 0)


def create_nerf_mvs(args, pts_embedder=True, use_mvs=False, dir_embedder=True, device=None):
    """Same contract as models.create_nerf_mvs: returns
    (render_kwargs_train, render_kwargs_test, start, grad_vars).  N_importance > 0 creates `network_fine` as the
    reference does (an MLP `rendering` ignores; its parameters join grad_vars).  When `args` has a `t_stop` attribute that is not
    None, both kwargs dicts also carry it, so `rendering(args, ..., **render_kwargs)` runs with early ray termination
    (see rendering); otherwise the dicts are exactly the reference's."""
    if not pts_embedder or dir_embedder:
        raise RuntimeError("create_nerf_mvs: the fused kernel implements pts_embedder=True, dir_embedder=False "
                           "(the combination every shipped caller uses)")
    if device is None:
        if not torch.cuda.is_available():
            raise RuntimeError("create_nerf_mvs: no CUDA device; mvsnerf_b200 has no CPU path")
        device = torch.device("cuda", torch.cuda.current_device())
    model = MVSNeRF(D=args.netdepth, W=args.netwidth, input_ch_pts=args.pts_dim * (1 + 2 * args.multires),
                    input_ch_views=args.dir_dim, input_ch_feat=args.feat_dim, net_type=args.net_type).to(device)
    grad_vars = list(model.parameters())
    model_fine = None
    if getattr(args, "N_importance", 0) > 0:
        # models.py:593-598: a second MLP whose parameters join grad_vars; `rendering` never runs it (nor does the
        # reference's), the importance samples are drawn from the density grid (build_density / ray_marcher_fine)
        model_fine = MVSNeRF(D=args.netdepth, W=args.netwidth, input_ch_pts=args.pts_dim * (1 + 2 * args.multires),
                             input_ch_views=args.dir_dim, input_ch_feat=args.feat_dim).to(device)
        grad_vars += list(model_fine.parameters())
    encoding_net = None
    if use_mvs:
        encoding_net = MVSNet().to(device)
        # models.py:622 adds the encoder's parameters here; this encoder is forward-only (no gradients reach it,
        # see MVSNet.forward), so handing them to the optimiser would only pretend to train them.
    ckpt_path = getattr(args, "ckpt", None)
    if ckpt_path is not None and ckpt_path != "None":
        ckpt = torch.load(ckpt_path, map_location=device, weights_only=False)
        if use_mvs:
            encoding_net.load_state_dict(ckpt["network_mvs_state_dict"])
        model.load_state_dict(ckpt["network_fn_state_dict"])
    render_kwargs_train = {
        "network_query_fn": lambda pts, viewdirs, rays_feats, network_fn: _network_query(
            pts, viewdirs, rays_feats, network_fn, args.netchunk),
        "perturb": args.perturb, "N_importance": args.N_importance, "network_fine": model_fine,
        "N_samples": args.N_samples, "network_fn": model, "network_mvs": encoding_net,
        "use_viewdirs": args.use_viewdirs, "white_bkgd": args.white_bkgd, "raw_noise_std": args.raw_noise_std,
    }
    if getattr(args, "t_stop", None) is not None:
        render_kwargs_train["t_stop"] = float(args.t_stop)
    render_kwargs_test = dict(render_kwargs_train)
    render_kwargs_test["perturb"] = False
    return render_kwargs_train, render_kwargs_test, 0, grad_vars


def load_weights_npz(model_fn: MVSNeRF | None, model_mvs: MVSNet | None, path: str):
    """Load the `mlp/` and `mvs/` tensors of tests/golden/mvsnerf_v0_weights.npz (an export of
    ckpts/mvsnerf-v0.tar that travels with the repository)."""
    import numpy as np
    z = np.load(path)
    if model_fn is not None:
        model_fn.load_state_dict({k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("mlp/")})
    if model_mvs is not None:
        model_mvs.load_state_dict({k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("mvs/")})
