"""H100 drop-ins for the reference's model API (SURVEY.md 8(b), "B-model").

`RADNeRF` / `RADNeRFTorso` here mirror modules/radnerfs/radnerf.py:13 and modules/radnerfs/radnerf_torso.py:17:
  * same constructor argument (the hparams dict), same parameter / buffer names and shapes, so
    `load_ckpt(model, dir, strict=True)` (utils/commons/ckpt_utils.py:29-76) and `.to(device).eval()` work;
  * same `render(rays_o, rays_d, cond, bg_coords, poses, index, dt_gamma, bg_color, perturb, force_all_rays,
    max_steps, T_thresh, ..., **kwargs)` signature and result dict (renderer.py:286 / radnerf_torso.py:86),
    tolerant of every extra kwarg the driver passes (`staged`, `lm68`, all hparams keys);
  * same errors-as-exceptions behaviour.
Everything under `render` runs in the fused sm_90a kernels of libgfpp.so through the C-ABI (include/gfpp.h).
Only the tiny conditioning nets (AudioNet / AudioAttNet, cond_encoder.py:98-180: 5x204 -> 64) stay in PyTorch,
as SURVEY.md 8(a) a4 prescribes.

Training: `RADNeRF` in `.train()` mode runs the reference's training branch of `render` (renderer.py:319-339, 385-398) on libgfpp's
training ops (train_ops.py) and its differentiable field, `RADNeRF.forward` (gfpp.h section G: fused fp32 forward and backward
kernels), so `loss.backward()` reaches the MLP weights, both grid tables, the individual code and the conditioning nets.  The SR and
torso classes are inference only: their `render` raises NotImplementedError in training mode.  `RADNeRFTorso.forward_torso` is
differentiable in training mode (gfpp.h section H), so the torso training step can be assembled from it and the training ops
(README.md shows the recipe).

`render_clip` is the clip-level entry point (SURVEY.md 8(f) rank 1): a whole clip of poses + conditioning is
rendered by a handful of persistent-kernel launches with rays generated in-kernel and frames kept on device.
"""
import copy
import ctypes
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _capi, video
from .config import GridLayout, cascade_count


MLP_PRECISIONS = {"fp32": 0, "fp16": 1, "bf16x3": 2, "bf16": 3, "robust": 4}


# ------------------------------------------------------------------------------------------------ small modules
class _MLPWeights(nn.Module):
    """Parameter container with the reference's key layout `net.{i}.weight` (cond_encoder.py:183-195, bias-free)."""

    def __init__(self, dim_in, dim_out, dim_hidden, num_layers):
        super().__init__()
        self.net = nn.ModuleList([
            nn.Linear(dim_in if l == 0 else dim_hidden, dim_out if l == num_layers - 1 else dim_hidden, bias=False)
            for l in range(num_layers)])


class _GridParams(nn.Module):
    """`embeddings` + `offsets` exactly like GridEncoder (gridencoder/grid.py:98-143)."""

    def __init__(self, layout: GridLayout):
        super().__init__()
        self.layout = layout
        self.register_buffer("offsets", torch.from_numpy(layout.offsets.copy()))
        self.embeddings = nn.Parameter(torch.empty(layout.n_entries, layout.level_dim).uniform_(-1e-4, 1e-4))


class _AudioNet(nn.Module):
    """cond_encoder.py:98-143: four Conv1d(k=3, padding=1) with window-size dependent strides that shrink the window to one
    step, then two Linear layers.  Same parameter names; same supported sizes -- the reference's `win_size == [5, 8]` branch can
    never be taken, so 5 and 8 raise ValueError there and here."""
    STRIDES = {1: (1, 1, 1, 1), 2: (2, 1, 1, 1), 3: (2, 2, 1, 1), 4: (2, 2, 1, 1), 16: (2, 2, 2, 2)}

    def __init__(self, dim_in, dim_aud, win_size=1):
        super().__init__()
        if win_size not in self.STRIDES:
            raise ValueError("unsupported win_size")
        self.win_size = win_size
        st = self.STRIDES[win_size]
        self.encoder_conv = nn.Sequential(
            nn.Conv1d(dim_in, 32, 3, st[0], 1), nn.LeakyReLU(0.02, True), nn.Conv1d(32, 32, 3, st[1], 1), nn.LeakyReLU(0.02, True),
            nn.Conv1d(32, 64, 3, st[2], 1), nn.LeakyReLU(0.02, True), nn.Conv1d(64, 64, 3, st[3], 1), nn.LeakyReLU(0.02, True))
        self.encoder_fc1 = nn.Sequential(nn.Linear(64, 64), nn.LeakyReLU(0.02, True), nn.Linear(64, dim_aud))

    def forward(self, x):  # [b, t=win_size, c]
        if self.win_size == 1:
            # Conv1d(k=3, padding=1) on a length-1 sequence only ever sees its centre tap: y = W[:, :, 1] x + b.  Written as
            # plain fp32 matmuls (a handful of launches per clip) instead of per-sample im2col convolutions.
            x = x.reshape(x.shape[0], -1)
            for i in (0, 2, 4, 6):
                conv = self.encoder_conv[i]
                x = F.leaky_relu(F.linear(x, conv.weight[:, :, 1], conv.bias), 0.02)
            return self.encoder_fc1(x)
        # audio-window conditioning (deepspeech 16x29, esperanto): the strided stack as the reference runs it
        y = x.permute(0, 2, 1)
        for i in (0, 2, 4, 6):
            conv = self.encoder_conv[i]
            y = F.leaky_relu(F.conv1d(y, conv.weight, conv.bias, stride=conv.stride, padding=1), 0.02)
        return self.encoder_fc1(y.squeeze(-1))


class _AudioAttNet(nn.Module):
    """cond_encoder.py:146-180; also a batched variant over frames."""

    def __init__(self, dim, seq_len):
        super().__init__()
        self.seq_len, self.in_out_dim = seq_len, dim
        self.attentionConvNet = nn.Sequential(
            nn.Conv1d(dim, 16, 3, 1, 1), nn.LeakyReLU(0.02, True), nn.Conv1d(16, 8, 3, 1, 1), nn.LeakyReLU(0.02, True),
            nn.Conv1d(8, 4, 3, 1, 1), nn.LeakyReLU(0.02, True), nn.Conv1d(4, 2, 3, 1, 1), nn.LeakyReLU(0.02, True),
            nn.Conv1d(2, 1, 3, 1, 1), nn.LeakyReLU(0.02, True))
        self.attentionNet = nn.Sequential(nn.Linear(seq_len, seq_len), nn.Softmax(dim=1))

    def forward(self, x):  # [seq, c] -> [c]
        return self.forward_batched(x.unsqueeze(0))[0]

    def forward_batched(self, x):  # [T, seq, c] -> [T, c]
        y = x[..., :self.in_out_dim].permute(0, 2, 1)                          # [T,c,seq]
        for i in (0, 2, 4, 6, 8):                                              # Conv1d(k=3, padding=1) as three shifted matmuls
            conv = self.attentionConvNet[i]
            yp = F.pad(y, (1, 1))
            S = y.shape[-1]
            y = sum(torch.einsum("oc,tcs->tos", conv.weight[:, :, k], yp[:, :, k:k + S]) for k in range(3)) + conv.bias.view(1, -1, 1)
            y = F.leaky_relu(y, 0.02)
        y = self.attentionNet(y.reshape(-1, self.seq_len)).unsqueeze(-1)       # [T,seq,1]
        return torch.sum(y * x, dim=1)


# ------------------------------------------------------------------------------------------------ head model
class RADNeRF(nn.Module):
    has_torso = False
    forwards_eye_area = True   # renderer.py:308 passes eye_area_percent on; radnerf_torso.py:86-106 lets it fall into **kwargs

    def __init__(self, hparams):
        super().__init__()
        self.hparams = copy.deepcopy(hparams)
        hp = self.hparams
        if not hp.get("cuda_ray", True):
            raise NotImplementedError("only the cuda_ray path exists (as in the reference)")
        # --- NeRFRenderer.__init__ (modules/radnerfs/renderer.py:66-102)
        self.bound = hp["bound"]
        self.cascade = cascade_count(hp["bound"])
        self.grid_size = hp["grid_size"]
        self.density_scale = 1
        self.min_near = hp["min_near"]
        self.density_thresh = hp["density_thresh"]
        b = float(self.bound)
        aabb = torch.tensor([-b, -b / 2, -b, b, b / 2, b], dtype=torch.float32)
        self.register_buffer("aabb_train", aabb.clone())
        self.register_buffer("aabb_infer", aabb.clone())
        self.individual_embedding_num = hp["individual_embedding_num"]
        self.individual_embedding_dim = hp["individual_embedding_dim"]
        if self.individual_embedding_dim > 0:
            self.individual_embeddings = nn.Parameter(torch.randn(self.individual_embedding_num, self.individual_embedding_dim) * 0.1)
        self.register_buffer("density_grid", torch.zeros([self.cascade, self.grid_size ** 3]))
        self.register_buffer("density_bitfield", torch.zeros(self.cascade * self.grid_size ** 3 // 8, dtype=torch.uint8))
        self.register_buffer("step_counter", torch.zeros(16, 2, dtype=torch.int32))
        self.mean_density = 0
        self.iter_density = 0
        self.mean_count = 0
        self.local_step = 0
        # --- RADNeRF.__init__ (modules/radnerfs/radnerf.py:14-86)
        if hp["cond_type"] == "esperanto":
            self.cond_in_dim = 44
        elif hp["cond_type"] == "deepspeech":
            self.cond_in_dim = 29
        elif hp["cond_type"] == "idexp_lm3d_normalized":
            self.cond_in_dim = {"lm68": 68 * 3, "lm131": 131 * 3, "lm468": 468 * 3}[hp.get("nerf_keypoint_mode", "lm68")]
        else:
            raise NotImplementedError()
        self.cond_out_dim = hp["cond_out_dim"] // 2 * 2
        self.cond_win_size = hp["cond_win_size"]
        self.smo_win_size = hp["smo_win_size"]
        self.cond_prenet = _AudioNet(self.cond_in_dim, self.cond_out_dim, win_size=self.cond_win_size)
        # eye-blink conditioning of the SR-era configs (radnerf.py:40-47; SURVEY.md 8(f) rank 2): same parameter names
        self.add_eye_blink_cond = bool(hp.get("add_eye_blink_cond", False))
        if self.add_eye_blink_cond:
            self.eye_blink_dim = int(hp["eye_blink_dim"])
            self.blink_embedding = nn.Embedding(1, self.cond_out_dim // 2)
            self.blink_encoder = nn.Sequential(nn.Linear(self.cond_out_dim // 2, self.cond_out_dim // 2),
                                               nn.Linear(self.cond_out_dim // 2, self.eye_blink_dim))
        self.with_att = hp["with_att"]
        if self.with_att:
            self.cond_att_net = _AudioAttNet(self.cond_out_dim, self.smo_win_size)
        gt = {"tiledgrid": "tiled", "hashgrid": "hash"}[hp["grid_type"]]
        it = hp["grid_interpolation_type"]
        self.position_embedder = _GridParams(GridLayout(3, log2_hashmap_size=hp["log2_hashmap_size"], desired_resolution=hp["desired_resolution"] * self.bound, gridtype=gt, interpolation=it))
        self.ambient_coord_dim = hp["ambient_coord_dim"]
        self.ambient_net = _MLPWeights(32 + self.cond_out_dim, self.ambient_coord_dim, hp["hidden_dim_ambient"], hp["num_layers_ambient"])
        self.ambient_embedder = _GridParams(GridLayout(self.ambient_coord_dim, log2_hashmap_size=hp["log2_hashmap_size"], desired_resolution=hp["desired_resolution"], gridtype=gt, interpolation=it))
        self.geo_feat_dim = hp["geo_feat_dim"]
        self.sigma_net = _MLPWeights(32 + 32, 1 + self.geo_feat_dim, hp["hidden_dim_sigma"], hp["num_layers_sigma"])
        self.color_net = _MLPWeights(16 + self.geo_feat_dim + self.individual_embedding_dim, 3, hp["hidden_dim_color"], hp["num_layers_color"])
        shape_ok = (hp["hidden_dim_ambient"] == 128 and hp["num_layers_ambient"] == 3 and hp["hidden_dim_sigma"] == 128 and
                    hp["num_layers_sigma"] == 3 and hp["geo_feat_dim"] == 128 and hp["hidden_dim_color"] == 128 and
                    hp["num_layers_color"] == 2 and self.cond_out_dim == 64 and self.ambient_coord_dim in (2, 3))
        if not shape_ok:
            raise NotImplementedError("libgfpp kernels are built for the May architecture (hidden 128, 3/3/2 layers, cond 64)")
        # arithmetic of the head MLP GEMMs (gfpp_model_desc.mlp_precision): "fp32" (CUDA-core FFMA), "fp16" (wgmma, what the
        # reference runs under autocast), "bf16x3" (wgmma hi/lo split, ~fp32 accuracy), "bf16" (wgmma), "robust" (wgmma fp16
        # with the hi/lo split on the ambient net only + a 16-bit fixed-point position table: holds 1e-3 on well-conditioned scenes)
        self.mlp_precision = hparams.get("gfpp_mlp_precision", "fp32")
        # arithmetic of the training field (forward() and the training branch of render()): "fp32" (CUDA-core FFMA, gfpp.h section
        # G) or "fp16" (fp16 wgmma operands, fp32 accumulation, fp32 parameters and gradients, section J: what the reference's
        # amp: true trains with, here without rounding the tables or the inputs of tanh and exp)
        self.train_precision = hparams.get("gfpp_train_precision", "fp32")
        self._packed = None  # (key, packed_dev, Model, keepalive)
        self._workspace = None

    # ------------------------------------------------------------------ state invalidation
    def _apply(self, fn, *a, **k):
        self._packed = None
        self._workspace = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._packed = None
        return super().load_state_dict(*a, **k)

    def invalidate(self):
        """Call after mutating parameters in place (the packed, transposed copies are rebuilt lazily)."""
        self._packed = None

    # ------------------------------------------------------------------ conditioning (plumbing, PyTorch)
    def cal_cond_feat(self, cond, eye_area_percent=None):
        """radnerf.py:88-106.  cond: [smo_win, 1, C] -> [64]."""
        # fp32 end to end: no autocast, no TF32 convolutions (the 1e-3 parity bar is against the fp32 oracle)
        with torch.autocast("cuda", enabled=False):
            feat = self.cond_prenet(cond.float())
            if self.add_eye_blink_cond:
                feat = self._add_blink(feat, eye_area_percent, 1)
            if self.with_att:
                feat = self.cond_att_net(feat)
        return feat

    def _add_blink(self, feat, eye_area_percent, n_frames):
        """radnerf.py:97-103: blink_encoder(blink_embedding[0] * eye_area_percent) is added to the first eye_blink_dim
        channels of EVERY row of the frame's window (zero-padded rows included); None means 0 %.  feat: [n_frames * S, C]
        (S window rows per frame, frame-major) or [S, C] for one frame; eye_area_percent: scalar / [n_frames]."""
        E = self.eye_blink_dim
        if eye_area_percent is None:
            pct = torch.zeros(n_frames, 1, device=feat.device, dtype=feat.dtype)
        else:
            pct = torch.as_tensor(eye_area_percent, device=feat.device, dtype=feat.dtype).reshape(n_frames, 1)
        blink = self.blink_encoder(self.blink_embedding.weight[0].reshape(1, -1) * pct)        # [n_frames, E]
        rows = feat.shape[0] // n_frames
        out = feat.clone()
        out[:, :E] = feat[:, :E] + blink.repeat_interleave(rows, dim=0)
        return out

    def cal_cond_feat_clip(self, cond_seq, eye_area_percent=None):
        """All frames at once: cond_seq [T,cond_win_size,C] ([T,1,204] for the May configs) -> [T,64]; windows as get_audio_features(att_mode=2)
        (modules/radnerfs/utils.py:86-102: centred, zero-padded).  eye_area_percent: [T] (add_eye_blink_cond models)."""
        with torch.autocast("cuda", enabled=False):
            T = cond_seq.shape[0]
            S = self.smo_win_size
            left = S // 2
            x = cond_seq.float().reshape(T, -1)
            pad = torch.zeros(left, x.shape[1], device=x.device, dtype=x.dtype)
            padr = torch.zeros(S - left - 1, x.shape[1], device=x.device, dtype=x.dtype)
            xp = torch.cat([pad, x, padr], 0)
            idx = torch.arange(T, device=x.device).unsqueeze(1) + torch.arange(S, device=x.device).unsqueeze(0)
            wins = xp[idx]                                                  # [T,S,C]
            feat = self.cond_prenet(wins.reshape(T * S, self.cond_win_size, -1))
            if self.add_eye_blink_cond:
                feat = self._add_blink(feat, eye_area_percent, T)
            feat = feat.view(T, S, -1)
            # the reference zero-pads the *window*, and the prenet maps a zero row to f(0) != 0: same here
            if self.with_att:
                feat = self.cond_att_net.forward_batched(feat)
            else:
                feat = feat[:, left]
        return feat

    # ------------------------------------------------------------------ packing
    def _grid_desc(self, gp: _GridParams, keep):
        lay = gp.layout
        d = _capi.GridDesc()
        emb = gp.embeddings.detach()
        if emb.dtype != torch.float32 or not emb.is_contiguous():
            emb = emb.float().contiguous()
        keep.append(emb)
        off = np.ascontiguousarray(gp.offsets.detach().cpu().numpy().astype(np.int32))
        keep.append(off)
        d.embeddings = emb.data_ptr()
        d.offsets_host = off.ctypes.data
        d.input_dim = lay.input_dim
        d.num_levels = lay.num_levels
        d.base_resolution = lay.base_resolution
        d.log2_per_level_scale = float(lay.S)
        d.gridtype = lay.gridtype_id
        d.interp = lay.interp_id
        d.align_corners = int(lay.align_corners)
        return d

    def _w(self, t, keep):
        t = t.detach()
        if t.dtype != torch.float32 or not t.is_contiguous():
            t = t.float().contiguous()
        keep.append(t)
        return t.data_ptr()

    def _fill_desc(self, d, keep):
        d.position_grid = self._grid_desc(self.position_embedder, keep)
        d.ambient_grid = self._grid_desc(self.ambient_embedder, keep)
        for i in range(3):
            d.ambient_w[i] = self._w(self.ambient_net.net[i].weight, keep)
            d.sigma_w[i] = self._w(self.sigma_net.net[i].weight, keep)
        for i in range(2):
            d.color_w[i] = self._w(self.color_net.net[i].weight, keep)
        d.cond_dim = self.cond_out_dim
        d.ind_dim = self.individual_embedding_dim
        if self.individual_embedding_dim > 0:
            # eval uses individual_embeddings[0] (renderer.py:313-315)
            d.individual_code = self._w(self.individual_embeddings[0], keep)
        bf = self.density_bitfield
        keep.append(bf)
        d.density_bitfield = bf.data_ptr()
        aabb = self.aabb_infer.detach().cpu().tolist()
        for i in range(6):
            d.aabb[i] = aabb[i]
        d.bound = float(self.bound)
        d.min_near = float(self.min_near)
        d.cascade = self.cascade
        d.grid_size = self.grid_size
        d.density_scale = float(self.density_scale)
        d.has_torso = 0
        d.mlp_precision = MLP_PRECISIONS[self.mlp_precision]

    def _head_pack_sources(self):
        """Every tensor of the head field that _fill_desc reads.  The pack holds transposed, rounded or folded copies of them (the
        colour-L0 bias folds individual_embeddings[0], the sigma-L2 geo rows fold into colour L0), so an in-place edit of any one
        must rebuild it."""
        ts = [self.density_bitfield, self.aabb_infer, self.position_embedder.embeddings, self.ambient_embedder.embeddings]
        ts += [l.weight for net in (self.ambient_net, self.sigma_net, self.color_net) for l in net.net]
        if self.individual_embedding_dim > 0:
            ts.append(self.individual_embeddings)
        return ts

    def _torso_pack_sources(self):
        """The tensors of the torso part of the pack (none for a head-only pack)."""
        return []

    def _ensure_packed(self, head_only=False):
        """The packed model, rebuilt when anything it was packed from has changed.  head_only: the caller reads only the head
        field (frozen_head), so a pack whose torso part is out of date still serves it; the torso training steps update the torso
        weights in place every step and would otherwise repack the head with each one."""
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppError("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        # in-place edits bump tensor._version, and a replaced tensor has a new data_ptr: either rebuilds the packed copies
        def vers(ts):
            return tuple((t.data_ptr(), int(t._version)) for t in ts)
        key = ((float(self.density_scale), dev.index, self.mlp_precision, vers(self._head_pack_sources())),
               (getattr(self, "mean_density_torso", None), vers(self._torso_pack_sources())))
        if self._packed is not None and (self._packed[0] == key or (head_only and self._packed[0][0] == key[0])):
            return self._packed
        L = _capi.lib()
        with torch.cuda.device(dev):
            _capi.check(L.gfpp_check_device(), "gfpp_check_device")
            keep = []
            d = _capi.ModelDesc()
            self._fill_desc(d, keep)
            nbytes = L.gfpp_model_packed_bytes(ctypes.byref(d))
            packed = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            model = _capi.Model()
            _capi.check(L.gfpp_model_pack(ctypes.byref(d), packed.data_ptr(), nbytes, ctypes.byref(model), _capi.stream_ptr(dev)),
                        "gfpp_model_pack")
        self._packed = (key, packed, model, keep)
        return self._packed

    # ------------------------------------------------------------------ core call
    def render_frames(self, cond_feat, *, rays_o=None, rays_d=None, poses_c2w=None, intrinsics=None, H=None, W=None,
                      pose6=None, bg_coords=None, bg_color=None, dt_gamma=0.0, max_steps=1024, T_thresh=1e-4,
                      want_torso_maps=True, want_stats=False, rgb_out=None, u8_out=None, want_aux=True, noise=None, alpha_out=None,
                      rgba_out=None):
        """Render F frames with one call into libgfpp.  Returns a dict of device tensors with a leading F axis.

        Either (rays_o, rays_d) [F,N,3] or (poses_c2w [F,4,4], intrinsics, H, W) must be given.
        noise: optional fp32 [F,N] (any shape of F*N values) in [0,1) on the model's device: jittered ray starts, ray i of frame f
        begins marching at near + clamp(near*dt_gamma, dt_min, dt_max) * noise[f,i] (the first-round `noises` of the reference's
        march_rays, raymarching.py:388-392).  None = start at near, as perturb=False does.
        rgb_out: optional contiguous fp32 [F,N,3] device view the kernel writes `rgb_map` into (e.g. a slice of the clip buffer:
        no copy afterwards); u8_out: optional contiguous uint8 [F,N,3] view that receives the video frame `(rgb*255).int()`
        straight from the epilogue kernel -- with u8_out and no rgb_out no fp32 frame is written at all.
        The frame's alpha matte, written by the same kernel and independent of bg_color (include/gfpp.h, gfpp_outputs): alpha_out,
        optional contiguous fp32 [F,N] view, receives the coverage A = weights_sum + (1 - weights_sum) * torso_alpha (result key
        `alpha_map`); rgba_out, optional contiguous uint8 [F,N,4] view (4-byte aligned), receives the premultiplied colour P as
        (P*255).int() in the first three bytes and (A*255).int() in the fourth (result key `rgba_u8`).  P + (1 - A) * B is the frame
        over a background B.  rgba_out alone is a complete call: no RGB frame is written then.
        want_aux=False skips the depth / weights_sum result tensors (they stay in the workspace)."""
        if self.training:
            raise NotImplementedError("libgfpp implements the inference branch only (renderer.py:340-384)")
        dev = self.density_bitfield.device
        L = _capi.lib()
        f32 = torch.float32
        cond_feat = cond_feat.to(dev, f32).reshape(-1, self.cond_out_dim).contiguous()
        Fn = cond_feat.shape[0]
        fr = _capi.Frames()
        hold = [cond_feat]
        if rays_o is not None:
            if rays_d is None or rays_d.numel() != rays_o.numel() or rays_o.numel() % (3 * Fn):
                raise ValueError(f"rays_o / rays_d must both be [{Fn},N,3]")
            rays_o = rays_o.to(dev, f32).reshape(Fn, -1, 3).contiguous()
            rays_d = rays_d.to(dev, f32).reshape(Fn, -1, 3).contiguous()
            N = rays_o.shape[1]
            fr.rays_o, fr.rays_d = rays_o.data_ptr(), rays_d.data_ptr()
            hold += [rays_o, rays_d]
        else:
            if poses_c2w is None or poses_c2w.numel() != Fn * 16:
                raise ValueError(f"poses_c2w must be [{Fn},4,4] (one pose per conditioning row)")
            poses_c2w = poses_c2w.to(dev, f32).reshape(Fn, 16).contiguous()
            N = H * W
            fr.poses_c2w = poses_c2w.data_ptr()
            fr.fx, fr.fy, fr.cx, fr.cy = [float(v) for v in intrinsics]
            fr.img_h, fr.img_w = H, W
            hold.append(poses_c2w)
        fr.n_frames, fr.n_rays = Fn, N
        fr.cond_feat = cond_feat.data_ptr()
        if self.has_torso:
            if pose6 is None or pose6.numel() != Fn * 6:
                raise ValueError(f"pose6 must be [{Fn},6]")
            if bg_coords is None or bg_coords.numel() != N * 2:
                raise ValueError(f"bg_coords must be [{N},2] (one row per ray)")
            pose6 = pose6.to(dev, f32).reshape(Fn, 6).contiguous()
            bg_coords = bg_coords.to(dev, f32).reshape(N, 2).contiguous()
            fr.torso_pose6, fr.bg_coords = pose6.data_ptr(), bg_coords.data_ptr()
            hold += [pose6, bg_coords]
        if bg_color is not None:
            if not torch.is_tensor(bg_color):
                bg_color = torch.full((N, 3), float(bg_color), device=dev, dtype=f32)
            bg_color = bg_color.to(dev, f32).reshape(-1, 3)
            if bg_color.shape[0] == 1:
                bg_color = bg_color.expand(N, 3)
            elif bg_color.shape[0] != N:
                raise ValueError(f"bg_color must have 1 or {N} rows (one per ray, shared by all frames), got {bg_color.shape[0]}")
            bg_color = bg_color.contiguous()
            fr.bg_color = bg_color.data_ptr()
            hold.append(bg_color)
        fr.dt_gamma, fr.max_steps, fr.T_thresh = float(dt_gamma), int(max_steps), float(T_thresh)
        if noise is not None:
            if not torch.is_tensor(noise) or noise.numel() != Fn * N:
                raise ValueError(f"noise must hold {Fn}*{N} values (one per ray and frame)")
            noise = noise.to(dev, f32).reshape(Fn, N).contiguous()
            fr.noises = noise.data_ptr()
            hold.append(noise)

        out = _capi.Outputs()
        res = {}
        if rgb_out is not None:
            if rgb_out.dtype != f32 or not rgb_out.is_contiguous() or rgb_out.numel() != Fn * N * 3 or rgb_out.device != dev:
                raise ValueError(f"rgb_out must be a contiguous fp32 [{Fn},{N},3] tensor on {dev}")
            res["rgb_map"] = rgb_out.view(Fn, N, 3)
        elif u8_out is None and rgba_out is None:
            res["rgb_map"] = torch.empty(Fn, N, 3, device=dev, dtype=f32)
        if u8_out is not None:
            if u8_out.dtype != torch.uint8 or not u8_out.is_contiguous() or u8_out.numel() != Fn * N * 3 or u8_out.device != dev:
                raise ValueError(f"u8_out must be a contiguous uint8 [{Fn},{N},3] tensor on {dev}")
            res["rgb_u8"] = u8_out.view(Fn, N, 3)
            out.rgb_u8 = u8_out.data_ptr()
        if alpha_out is not None:
            if alpha_out.dtype != f32 or not alpha_out.is_contiguous() or alpha_out.numel() != Fn * N or alpha_out.device != dev:
                raise ValueError(f"alpha_out must be a contiguous fp32 [{Fn},{N}] tensor on {dev}")
            res["alpha_map"] = alpha_out.view(Fn, N)
            out.alpha_map = alpha_out.data_ptr()
        if rgba_out is not None:
            if (rgba_out.dtype != torch.uint8 or not rgba_out.is_contiguous() or rgba_out.numel() != Fn * N * 4 or rgba_out.device != dev
                    or rgba_out.data_ptr() % 4):
                raise ValueError(f"rgba_out must be a contiguous, 4-byte aligned uint8 [{Fn},{N},4] tensor on {dev}")
            res["rgba_u8"] = rgba_out.view(Fn, N, 4)
            out.rgba_u8 = rgba_out.data_ptr()
        if "rgb_map" in res:
            out.rgb_map = res["rgb_map"].data_ptr()
        if want_aux:
            res["depth_map"] = torch.empty(Fn, N, device=dev, dtype=f32)
            res["weights_sum"] = torch.empty(Fn, N, device=dev, dtype=f32)
            out.depth_map, out.weights_sum = res["depth_map"].data_ptr(), res["weights_sum"].data_ptr()
        if self.has_torso and want_torso_maps:
            res["torso_alpha_map"] = torch.empty(Fn, N, device=dev, dtype=f32)
            res["torso_rgb_map"] = torch.empty(Fn, N, 3, device=dev, dtype=f32)
            res["deform"] = torch.empty(Fn, N, 2, device=dev, dtype=f32)
            out.torso_alpha_map, out.torso_rgb_map, out.torso_deform = (res["torso_alpha_map"].data_ptr(), res["torso_rgb_map"].data_ptr(), res["deform"].data_ptr())
        if want_stats:
            res["stats"] = torch.empty(Fn, 4, device=dev, dtype=torch.int32)
            out.stats = res["stats"].data_ptr()
        _, packed, model, _keep = self._ensure_packed()   # after the argument checks: a bad call launches nothing
        need = L.gfpp_render_workspace_bytes(Fn, N, int(max_steps))
        if self._workspace is None or self._workspace.numel() < need or self._workspace.device != dev:
            self._workspace = torch.empty(need, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _capi.check(L.gfpp_render_frames(ctypes.byref(model), ctypes.byref(fr), ctypes.byref(out), self._workspace.data_ptr(),
                                             self._workspace.numel(), _capi.stream_ptr(dev)), "gfpp_render_frames")
        self.last_launch_count = int(L.gfpp_last_launch_count())
        del hold
        return res

    def generate_rays(self, poses_c2w, intrinsics, H, W):
        """The rays the clip path generates in-kernel, written out (debug / tests): ([F,H*W,3], [F,H*W,3]) on the model's device."""
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppError("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        poses = poses_c2w.to(dev, torch.float32).reshape(-1, 16).contiguous()
        Fn = poses.shape[0]
        ro = torch.empty(Fn, H * W, 3, device=dev, dtype=torch.float32)
        rd = torch.empty_like(ro)
        fx, fy, cx, cy = [float(v) for v in intrinsics]
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_debug_generate_rays(poses.data_ptr(), Fn, fx, fy, cx, cy, H, W, ro.data_ptr(), rd.data_ptr(),
                                                           _capi.stream_ptr(dev)), "gfpp_debug_generate_rays")
        return ro, rd

    # ------------------------------------------------------------------ occupancy grid (NeRFRenderer, renderer.py:117-284)
    @torch.no_grad()
    def density(self, position, cond_feat, e=None, cond_mask=None):
        """radnerf.py:143-166: {'sigma': trunc_exp(h0) [N], 'geo_feat': h[1:129] [N,128]} for positions [N,3] in [-bound, bound]
        and one conditioning vector [64].  libgfpp evaluates the field of the model's mode: fp16 models on wgmma with their fp16
        operand images and tables, the other modes in fp32."""
        _, _, model, _ = self._ensure_packed()
        dev = self.density_bitfield.device
        x = position.to(dev, torch.float32).reshape(-1, 3).contiguous()
        c = cond_feat.to(dev, torch.float32).reshape(-1).contiguous()
        if c.numel() != self.cond_out_dim:
            raise ValueError(f"density() takes one conditioning vector of {self.cond_out_dim} values")
        n = x.shape[0]
        sigma = torch.empty(n, device=dev, dtype=torch.float32)
        geo = torch.empty(n, self.geo_feat_dim, device=dev, dtype=torch.float32)
        if n:
            with torch.cuda.device(dev):
                _capi.check(_capi.lib().gfpp_density_query(ctypes.byref(model), x.data_ptr(), n, c.data_ptr(), sigma.data_ptr(),
                                                           geo.data_ptr(), _capi.stream_ptr(dev)), "gfpp_density_query")
        return {"sigma": sigma, "geo_feat": geo}

    def reset_extra_state(self):
        """renderer.py:117-129."""
        self.density_grid.zero_()
        self.mean_density = 0
        self.iter_density = 0
        self.step_counter.zero_()
        self.mean_count = 0
        self.local_step = 0

    def _cell_noise(self, S, dev):
        """The reference's rand_like draws (renderer.py:238-258) as one [C,H,H,H,3] tensor: chunks of S cells per axis, x-major,
        one [chunk, 3] draw per cascade inside each chunk."""
        H, C = self.grid_size, self.cascade
        if S >= H:
            return torch.stack([torch.rand(H ** 3, 3, device=dev) for _ in range(C)]).view(C, H, H, H, 3)
        noise = torch.empty(C, H, H, H, 3, device=dev)
        for x0 in range(0, H, S):
            for y0 in range(0, H, S):
                for z0 in range(0, H, S):
                    nx, ny, nz = min(S, H - x0), min(S, H - y0), min(S, H - z0)
                    for cas in range(C):
                        noise[cas, x0:x0 + nx, y0:y0 + ny, z0:z0 + nz] = torch.rand(nx * ny * nz, 3, device=dev).view(nx, ny, nz, 3)
        return noise

    def refresh_density_grid(self, cond_feat, noise, decay=0.95, tmp_grid=None):
        """The device half of update_extra_state (renderer.py:230-278) in libgfpp, on the current stream, no host sync:
        density_grid (EMA, in place), the bitfield and the packed model's derived occupancy.  Returns the device scalar
        mean_density.  tmp_grid: optional [C, H^3] fp32 tensor that receives the raw (pre-dilation) densities."""
        _, _, model, _ = self._ensure_packed()
        dev = self.density_bitfield.device
        L = _capi.lib()
        C, H = self.cascade, self.grid_size
        c = cond_feat.to(dev, torch.float32).reshape(-1).contiguous()
        if c.numel() != self.cond_out_dim:
            raise ValueError(f"the grid refresh takes one conditioning vector of {self.cond_out_dim} values")
        noise = noise.to(dev, torch.float32).contiguous()
        if noise.numel() != C * H ** 3 * 3:
            raise ValueError(f"noise must be [{C},{H},{H},{H},3]")
        g = self.density_grid
        if g.dtype != torch.float32 or not g.is_contiguous():
            raise ValueError("density_grid must be a contiguous fp32 buffer")
        if tmp_grid is not None and (tmp_grid.dtype != torch.float32 or not tmp_grid.is_contiguous() or tmp_grid.numel() != C * H ** 3
                                     or tmp_grid.device != dev):
            raise ValueError(f"tmp_grid must be a contiguous fp32 [{C},{H ** 3}] tensor on {dev}")
        need = L.gfpp_density_grid_workspace_bytes(C, H)
        if need == 0:
            raise _capi.GfppError(f"the grid refresh does not support cascade {C} / grid_size {H}")
        ws = self.__dict__.get("_grid_ws")
        if ws is None or ws.numel() < need or ws.device != dev:
            ws = self.__dict__["_grid_ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
        mean = torch.empty(1, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            # writes density_bitfield through its pointer: its _version does not move, so the packed model stays valid (the
            # call itself rebuilt the packed occupancy bounds and coarse bits)
            _capi.check(L.gfpp_density_grid_update(ctypes.byref(model), c.data_ptr(), noise.data_ptr(), float(decay), float(self.density_thresh),
                                                   g.data_ptr(), mean.data_ptr(), None if tmp_grid is None else tmp_grid.data_ptr(),
                                                   ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_density_grid_update")
        self.last_launch_count = int(L.gfpp_last_launch_count())
        return mean

    @torch.no_grad()
    def update_extra_state(self, decay=0.95, S=128, *, cond_index=None, noise=None):
        """renderer.py:201-284 (the to_heatmap branch is not supported, as in the reference's own density()).  The conditioning
        window comes from `self.conds` at `cond_index` (default: random.randint, as the reference) and the cell jitter from
        `noise` [C,H,H,H,3] in [0,1) (default: torch.rand in the reference's draw order for chunk size S)."""
        import random
        from .scene import cond_window
        if self.hparams.get("to_heatmap", False):
            raise NotImplementedError("to_heatmap: the reference's density() asserts against it (radnerf.py:147)")
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppError("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        if cond_index is None:
            cond_index = random.randint(0, self.conds.shape[0] - 1)
        cond = cond_window(self.conds, cond_index, self.smo_win_size).to(dev)
        cond_feat = self.cal_cond_feat(cond)
        if noise is None:
            noise = self._cell_noise(S, dev)
        mean = self.refresh_density_grid(cond_feat, noise, decay)
        self.mean_density = mean.item()
        self.iter_density += 1
        total_step = min(16, self.local_step)
        if total_step > 0:
            self.mean_count = int(self.step_counter[:total_step, 0].sum().item() / total_step)
        self.local_step = 0

    @torch.no_grad()
    def mark_untrained_grid(self, poses, intrinsic, S=64):
        """renderer.py:131-199: cells of density_grid that no camera of poses [B,4,4] (c2w) sees become -1.  intrinsic =
        (fx, fy, cx, cy), taken as Python floats like the reference.  S (the reference's chunk size) does not change the result."""
        dev = self.density_grid.device
        if dev.type != "cuda":
            raise _capi.GfppError("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        if isinstance(poses, np.ndarray):
            poses = torch.from_numpy(poses)
        P = poses.to(dev, torch.float32).reshape(-1, 16).contiguous()
        fx, fy, cx, cy = [float(v) for v in intrinsic]
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_mark_untrained_grid(P.data_ptr(), P.shape[0], fx, fy, cx, cy, float(self.bound), self.cascade,
                                                             self.grid_size, self.density_grid.data_ptr(), _capi.stream_ptr(dev)),
                        "gfpp_mark_untrained_grid")

    # ------------------------------------------------------------------ the differentiable field (training)
    def forward(self, position, direction, cond_feat, individual_code, cond_mask=None):
        """radnerf.py:108-141: (sigma [N] raw, color [N,3], ambient_pos [N,A]) at positions [N,3] in [-bound, bound] and directions
        [N,3], for one conditioning vector [1,64] and one individual code [ind_dim] (or None).  Differentiable w.r.t. the eight MLP
        weights, both grid tables, cond_feat and individual_code, through libgfpp's fused kernels: fp32 FFMA (gfpp.h section G) or,
        with train_precision = "fp16", fp16 tensor-core products with fp32 accumulation (section J).  cond_mask is accepted and
        ignored, as in the reference.  Parameters, outputs and gradients are fp32 in both, also under torch.autocast, which does not
        reach into the field (with train_precision = "fp32" that is the reference's amp: false arithmetic)."""
        if self.mlp_precision != "fp32":
            raise NotImplementedError(f"the training field runs in fp32 only (mlp_precision is {self.mlp_precision!r})")
        if self.train_precision not in ("fp32", "fp16"):
            raise ValueError(f'train_precision must be "fp32" or "fp16", got {self.train_precision!r}')
        if position.requires_grad or direction.requires_grad:
            raise NotImplementedError("gradients w.r.t. positions or directions (camera-pose optimisation) are not implemented")
        if self.density_bitfield.device.type != "cuda":
            raise _capi.GfppNoCpuPath("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        from . import train_ops
        params = ([self.ambient_net.net[i].weight for i in range(3)] + [self.sigma_net.net[i].weight for i in range(3)] +
                  [self.color_net.net[i].weight for i in range(2)] + [self.position_embedder.embeddings, self.ambient_embedder.embeddings])
        code = individual_code if self.individual_embedding_dim > 0 else None
        with torch.autocast("cuda", enabled=False):
            return train_ops.field(self, position, direction, cond_feat, code, *params)

    def _render_train(self, rays_o, rays_d, cond, index, dt_gamma, bg_color, perturb, force_all_rays, max_steps, cond_mask, eye_area_percent):
        """The training branch of renderer.py:286-339 plus the shared tail 385-398."""
        from . import train_ops
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppNoCpuPath("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        prefix = rays_o.shape[:-1]
        rays_o = rays_o.to(dev).contiguous().view(-1, 3)
        rays_d = rays_d.to(dev).contiguous().view(-1, 3)
        nears, fars = train_ops.near_far_from_aabb(rays_o, rays_d, self.aabb_train, self.min_near)
        cond_feat = self.cal_cond_feat(cond.to(dev), eye_area_percent=eye_area_percent if self.forwards_eye_area else None)
        ind_code = self.individual_embeddings[index] if self.individual_embedding_dim > 0 else None
        counter = self.step_counter[self.local_step % 16]
        counter.zero_()
        self.local_step += 1
        xyzs, dirs, deltas, rays = train_ops.march_rays_train(rays_o, rays_d, self.bound, self.density_bitfield, self.cascade, self.grid_size, nears,
                                                              fars, counter, self.mean_count, perturb, 128, force_all_rays, dt_gamma, max_steps)
        sigmas, rgbs, ambient = self.forward(xyzs, dirs, cond_feat, ind_code, cond_mask=cond_mask)
        sigmas = self.density_scale * sigmas
        weights_sum, ambient_sum, depth, image = train_ops.composite_rays_train(sigmas, rgbs, ambient.abs().sum(-1), deltas, rays)
        results = {"weights_sum": weights_sum, "ambient": ambient_sum, "position": xyzs}
        if bg_color is None:
            bg_color = 1
        elif torch.is_tensor(bg_color):
            bg_color = bg_color.to(dev)
        image = image + (1 - weights_sum).unsqueeze(-1) * bg_color
        results["rgb_map"] = image.view(*prefix, 3).clamp(0, 1)
        results["depth_map"] = (torch.clamp(depth - nears, min=0) / (fars - nears)).view(*prefix)
        return results

    # ------------------------------------------------------------------ the frozen head of the torso training steps
    def _aabb_train_host(self):
        """aabb_train as six host floats, copied from the device once per buffer version (the slab test takes them by value)."""
        key = (self.aabb_train.data_ptr(), self.aabb_train._version)
        cached = self.__dict__.get("_aabb_train_cache")
        if cached is None or cached[0] != key:
            vals = (ctypes.c_float * 6)(*[float(v) for v in self.aabb_train.detach().cpu().tolist()])
            cached = self.__dict__["_aabb_train_cache"] = (key, vals)
        return cached[1]

    def frozen_head(self, rays_o, rays_d, cond_feat, ind_code, perturb=False, dt_gamma=0, max_steps=1024, T_thresh=1e-4, force_all_rays=False):
        """The no-grad head block of the torso training step (radnerf_torso.py:92-150, radnerf_torso_sr.py:150) in one fused pass over
        the packed head model (gfpp.h section K): (weights_sum [N], image [N,3]) fp32, the first and fourth outputs of
        near_far_from_aabb(aabb_train) + march_rays_train + forward + composite_rays_train, without ambient_sum and depth.

        rays_o / rays_d: [..., 3] with N rays.  cond_feat: one conditioning vector ([64] or [1,64]).  ind_code: the training row
        individual_embeddings[index] (a device tensor, read on the device), or None iff the model has no individual codes.  The
        head runs in the model's mlp_precision (fp32, or the arithmetic of the torso configs' amp: true with "fp16"), in train or
        eval mode, and never records autograd.  perturb=True draws one torch.rand(N) on the model's device before anything else
        random, as march_rays_train does, so a seeded call jitters each ray as the composed path does.  step_counter / local_step
        are neither read nor written; with mean_count > 0 march_rays_train would truncate rays to its sample budget, which this
        call does not model, so it raises unless force_all_rays."""
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppNoCpuPath("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        if not force_all_rays and self.mean_count > 0:
            raise ValueError(f"frozen_head: mean_count is {self.mean_count}: march_rays_train would cut rays to that sample budget "
                             "(pass force_all_rays=True to give every ray max_steps samples)")
        f32 = torch.float32
        if not torch.is_tensor(rays_o) or not torch.is_tensor(rays_d) or rays_o.shape[-1] != 3 or rays_o.shape != rays_d.shape or rays_o.numel() == 0:
            raise ValueError(f"rays_o and rays_d must both be [...,3] with the same shape, got {tuple(getattr(rays_o, 'shape', ()))} and "
                             f"{tuple(getattr(rays_d, 'shape', ()))}")
        if not torch.is_tensor(cond_feat) or cond_feat.numel() != self.cond_out_dim:
            raise ValueError(f"cond_feat must hold one conditioning vector of {self.cond_out_dim} values")
        dim = self.individual_embedding_dim
        if (ind_code is None) != (dim == 0) or (ind_code is not None and (not torch.is_tensor(ind_code) or ind_code.numel() != dim)):
            raise ValueError(f"ind_code must hold {dim} values (None iff the model has no individual codes)")
        if not 1 <= int(max_steps) <= 4096:
            raise ValueError(f"max_steps must be in 1..4096, got {max_steps}")
        N = rays_o.numel() // 3
        with torch.no_grad():
            noise = torch.rand(N, dtype=f32, device=dev) if perturb else None
            _, _, model, _ = self._ensure_packed(head_only=True)
            L = _capi.lib()
            ro = rays_o.detach().to(dev, f32).reshape(N, 3).contiguous()
            rd = rays_d.detach().to(dev, f32).reshape(N, 3).contiguous()
            c = cond_feat.detach().to(dev, f32).reshape(-1).contiguous()
            code = ind_code.detach().to(dev, f32).reshape(-1).contiguous() if ind_code is not None else None
            weights_sum = torch.empty(N, dtype=f32, device=dev)
            image = torch.empty(N, 3, dtype=f32, device=dev)
            need = L.gfpp_frozen_head_workspace_bytes(N, int(max_steps))
            if need == 0:
                raise _capi.GfppError(f"frozen_head does not support {N} rays")
            ws = self.__dict__.get("_frozen_ws")
            if ws is None or ws.numel() < need or ws.device != dev:
                ws = self.__dict__["_frozen_ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                _capi.check(L.gfpp_frozen_head(ctypes.byref(model), ro.data_ptr(), rd.data_ptr(), N, self._aabb_train_host(), c.data_ptr(),
                                               None if code is None else code.data_ptr(), None if noise is None else noise.data_ptr(),
                                               float(dt_gamma), int(max_steps), float(T_thresh), weights_sum.data_ptr(), image.data_ptr(),
                                               ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_frozen_head")
            self.last_launch_count = int(L.gfpp_last_launch_count())
        return weights_sum, image

    # ------------------------------------------------------------------ the reference's render()
    trains_field = True   # render() has a training branch; the SR and torso subclasses do not

    def render(self, rays_o, rays_d, cond, bg_coords, poses, index=0, dt_gamma=0, bg_color=None, perturb=False,
               force_all_rays=False, max_steps=1024, T_thresh=1e-4, cond_mask=None, eye_area_percent=None, **kwargs):
        """renderer.py:286-399.  In training mode: the differentiable training branch (T_thresh is not used there, as in the reference,
        which calls composite_rays_train with its default); otherwise the fused inference renderer, without autograd.  perturb=True
        outside training (the reference's validation_step) jitters each ray's start with one torch.rand(N) draw on the model's
        device, as the reference's first march_rays round does (_ray_start_noise)."""
        if self.training:
            if not self.trains_field:
                raise NotImplementedError(f"{type(self).__name__} renders for inference only; training covers the head field (RADNeRF)")
            return self._render_train(rays_o, rays_d, cond, index, dt_gamma, bg_color, perturb, force_all_rays, max_steps, cond_mask,
                                      eye_area_percent)
        with torch.no_grad():
            return self._render_eval(rays_o, rays_d, cond, bg_coords, poses, dt_gamma, bg_color, perturb, max_steps, T_thresh, cond_mask,
                                     eye_area_percent)

    def _ray_start_noise(self, n_rays):
        """perturb=True outside training (the reference's validation_step): the first round of renderer.py:354-384 passes
        `perturb` to march_rays, which draws torch.rand(n_alive) with all N rays alive (raymarching.py:388-390); later rounds pass
        False and draw nothing.  One draw of N values on the model's device, made before any later draw of the same call (the
        SR head's random noise planes), so a seeded call consumes the generator exactly as the reference does."""
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppNoCpuPath("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        return torch.rand(n_rays, dtype=torch.float32, device=dev)

    def _render_eval(self, rays_o, rays_d, cond, bg_coords, poses, dt_gamma, bg_color, perturb, max_steps, T_thresh, cond_mask, eye_area_percent):
        # perturb: jittered ray starts (_ray_start_noise); the jitter moves where each ray starts marching, nothing else
        # cond_mask: accepted and ignored, exactly like the reference -- its forward() / density() take the argument and never read
        # it (radnerf.py:108-141, 143-165); the only requirement renderer.py:371-372 puts on it is one entry per ray
        if cond_mask is not None and torch.is_tensor(cond_mask) and cond_mask.shape[0] != rays_o.numel() // 3:
            raise IndexError("cond_mask must have one entry per ray (renderer.py:372 indexes it with rays_alive)")
        prefix = rays_o.shape[:-1]
        if rays_o.numel() // 3 != int(np.prod(prefix)) or (len(prefix) > 1 and prefix[0] != 1):
            raise ValueError("render() assumes B == 1 (renderer.py:287)")
        cond_feat = self.cal_cond_feat(cond.to(self.density_bitfield.device),
                                       eye_area_percent=eye_area_percent if self.forwards_eye_area else None)
        noise = self._ray_start_noise(rays_o.numel() // 3) if perturb else None
        res = self.render_frames(cond_feat.reshape(1, -1), rays_o=rays_o.reshape(1, -1, 3), rays_d=rays_d.reshape(1, -1, 3),
                                 pose6=poses if self.has_torso else None, bg_coords=bg_coords if self.has_torso else None,
                                 bg_color=bg_color, dt_gamma=dt_gamma, max_steps=max_steps, T_thresh=T_thresh, noise=noise)
        results = {"depth_map": res["depth_map"].view(*prefix), "rgb_map": res["rgb_map"].view(*prefix, 3),
                   "weights_sum": res["weights_sum"].view(-1)}
        if self.has_torso:
            alpha = res["torso_alpha_map"].view(-1, 1)
            results["torso_alpha_map"] = alpha
            trgb = res["torso_rgb_map"].view(-1, 3)
            results["torso_rgb_map"] = trgb.view(1, -1, 3) if (bg_color is not None and torch.is_tensor(bg_color) and bg_color.dim() == 3) else trgb
            mask = self.torso_mask(bg_coords)
            if bool(mask.any()):
                results["deform"] = res["deform"].view(-1, 2)[mask]
        return results

    # ------------------------------------------------------------------ clip API
    @torch.no_grad()
    def render_clip(self, poses_c2w, intrinsics, H, W, cond_seq=None, cond_feat=None, bg_color=None, bg_coords=None, pose6=None,
                    dt_gamma=None, max_steps=None, T_thresh=1e-2, frames_per_call=64, out=None, want_stats=False,
                    eye_area_percent=None, as_uint8=False, as_rgba=False, as_yuv420=False):
        """Render a clip: poses_c2w [T,4,4], cond_seq [T,1,C] (or precomputed cond_feat [T,64]); eye_area_percent [T] for
        add_eye_blink_cond models.  Returns rgb [T,H*W,3] on the model's device: fp32 clamped to [0,1], or -- as_uint8 -- the
        uint8 video frames `(rgb*255).int()` (genefacepp_infer.py:469,505) written by the epilogue kernel itself, or -- as_rgba --
        uint8 [T,H*W,4] alpha-matte frames: premultiplied colour P and coverage A, each `(x*255).int()`, so that P + (1 - A) * B is
        the frame over any background B (render_frames' rgba_out), or -- as_yuv420 -- uint8 [T,H*W*3/2] planar I420 frames, the
        as_uint8 frames converted on the GPU (video.rgb_u8_to_i420; H and W must be even).  The matte is defined without a
        background: as_rgba with bg_color raises ValueError, as does asking for two of the three formats.  `out`: optional
        preallocated result buffer of that dtype and shape; every call writes its frames straight into it (as_yuv420: each call's
        uint8 frames go to a scratch buffer the model keeps, then are converted into `out`)."""
        if as_rgba and as_uint8:
            raise ValueError("as_rgba and as_uint8 are two different frame formats: pick one")
        if as_yuv420 and (as_uint8 or as_rgba):
            raise ValueError("as_yuv420 is a frame format of its own: it cannot be combined with as_uint8 or as_rgba")
        if as_rgba and bg_color is not None:
            raise ValueError("as_rgba returns the frame's matte, which does not depend on a background: composite P + (1 - A) * B "
                             "instead of passing bg_color")
        if as_yuv420:
            video.check_i420_size(H, W)
        dev = self.density_bitfield.device
        T = poses_c2w.shape[0]
        hp = self.hparams
        dt_gamma = hp["dt_gamma"] if dt_gamma is None else dt_gamma
        max_steps = hp["max_steps"] if max_steps is None else max_steps
        N = H * W
        odt = torch.uint8 if as_uint8 or as_rgba or as_yuv420 else torch.float32
        shape = (T, video.i420_frame_bytes(H, W)) if as_yuv420 else (T, N, 4 if as_rgba else 3)
        rgb = out if out is not None else torch.empty(shape, device=dev, dtype=odt)
        if rgb.dtype != odt or rgb.numel() != math.prod(shape) or not rgb.is_contiguous():
            raise ValueError(f"out must be a contiguous {odt} [{','.join(map(str, shape))}] tensor")
        rgb = rgb.view(shape)
        if cond_feat is None:
            cond_feat = self.cal_cond_feat_clip(cond_seq.to(dev), eye_area_percent=eye_area_percent if self.forwards_eye_area else None)
        poses_c2w = poses_c2w.to(dev, torch.float32)
        if self.has_torso and pose6 is None:
            from .scene import convert_poses
            pose6 = convert_poses(poses_c2w.cpu()).to(dev)
        dst = "rgba_out" if as_rgba else "u8_out" if as_uint8 or as_yuv420 else "rgb_out"
        stats = []
        for s in range(0, T, frames_per_call):
            e = min(T, s + frames_per_call)
            buf = video.frame_scratch(self, (e - s, N, 3)) if as_yuv420 else rgb[s:e]
            res = self.render_frames(cond_feat[s:e], poses_c2w=poses_c2w[s:e], intrinsics=intrinsics, H=H, W=W,
                                     pose6=pose6[s:e] if self.has_torso else None, bg_coords=bg_coords, bg_color=bg_color,
                                     dt_gamma=dt_gamma, max_steps=max_steps, T_thresh=T_thresh, want_torso_maps=False,
                                     want_stats=want_stats, want_aux=False, **{dst: buf})
            if as_yuv420:
                video.rgb_u8_to_i420(buf, H, W, out=rgb[s:e])
            if want_stats:
                stats.append(res["stats"])
        if want_stats:
            return rgb, torch.cat(stats, 0)
        return rgb


# ------------------------------------------------------------------------------------------------ head model + super-resolution
def _i420_out(out, T, S, dev):
    """The I420 result buffer [T,S*S*3/2] of an SR clip (S = 512): `out` checked, or a new one."""
    shape = (T, video.i420_frame_bytes(S, S))
    out = out if out is not None else torch.empty(shape, device=dev, dtype=torch.uint8)
    if out.shape != shape or out.dtype != torch.uint8 or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous uint8 [{T},{shape[1]}] tensor")
    return out


def _no_sr_matte(as_rgba):
    """The SR head is not linear in its input, so no alpha composes its 512x512 frame from the NeRF's matte: the SR models have
    no as_rgba output."""
    if as_rgba:
        raise ValueError("as_rgba is not available for the SR models: the SR head is not linear in its input, so no alpha matte "
                         "composes its 512x512 frame")


class RADNeRFwithSR(RADNeRF):
    """modules/radnerfs/radnerf_sr.py:50-210: the same head field rendered at 256x256 plus the `sr_net` 256 -> 512 head
    (genefaceplusplus_b200/superres.py).  Same extra state (`sr_net.*`, `lambda_ambient`) and result keys: `rgb_map` becomes
    the 256x256 image [1,3,256,256], `sr_rgb_map` the clamped 512x512 one (what the driver takes when `with_sr`,
    inference/genefacepp_infer.py:464-465, 480-481)."""
    sr_input_resolution = 256
    trains_field = False

    def __init__(self, hparams):
        super().__init__(hparams)
        from .superres import Superresolution
        self.sr_net = Superresolution(channels=3)
        self.lambda_ambient = nn.Parameter(torch.tensor([1.0]), requires_grad=False)

    def render(self, rays_o, rays_d, cond, bg_coords, poses, index=0, dt_gamma=0, bg_color=None, perturb=False,
               force_all_rays=False, max_steps=1024, T_thresh=1e-4, cond_mask=None, eye_area_percent=None, **kwargs):
        results = super().render(rays_o, rays_d, cond, bg_coords, poses, index, dt_gamma, bg_color, perturb, force_all_rays,
                                 max_steps, T_thresh, cond_mask, eye_area_percent=eye_area_percent, **kwargs)
        R = self.sr_input_resolution
        rgb_image = results["rgb_map"].reshape(1, R, R, 3).permute(0, 3, 1, 2)   # radnerf_sr.py:205 hard-codes 256 too
        with torch.autocast(rgb_image.device.type, enabled=False):
            sr = self.sr_net(rgb_image, noise_mode=kwargs.get("sr_noise_mode", "random")).clamp(0, 1)
        results["rgb_map"] = rgb_image
        results["sr_rgb_map"] = sr
        return results

    @torch.no_grad()
    def render_clip(self, poses_c2w, intrinsics, H=256, W=256, *args, sr_noise_mode="random", sr_frames_per_call=8, as_uint8=False,
                    as_rgba=False, as_yuv420=False, **kwargs):
        """Clip API: NeRF at 256x256 for all frames (libgfpp), then the SR head over chunks of frames.
        Returns the clamped 512x512 frames [T,3,512,512]; `intrinsics` are those of the 256x256 camera.
        as_uint8: returns the video frames uint8 [T,512,512,3] (HWC) `(rgb*255).int()` instead, written by the SR head's last
        kernel chunk by chunk into `out` (optional preallocated buffer of that shape); the NeRF stage still renders fp32, the
        SR head's input.  as_yuv420: the same frames as planar I420, uint8 [T,512*512*3/2] (video.rgb_u8_to_i420), each SR chunk's
        uint8 frames converted from a scratch buffer the model keeps into `out`; the noise planes are drawn as with as_uint8.
        Without either, `out` is the NeRF clip's buffer ([T,256*256,3] fp32), as in RADNeRF.render_clip.
        as_rgba raises ValueError (_no_sr_matte), and so does as_yuv420 with as_uint8."""
        _no_sr_matte(as_rgba)
        if as_yuv420 and as_uint8:
            raise ValueError("as_yuv420 is a frame format of its own: it cannot be combined with as_uint8 or as_rgba")
        from .dist import to_uint8
        R = self.sr_input_resolution
        if (H, W) != (R, R):
            raise ValueError(f"SR models render the NeRF at {R}x{R} (radnerf_sr.py:205)")
        want_stats = kwargs.get("want_stats", False)
        u8 = kwargs.pop("out", None) if as_uint8 or as_yuv420 else None
        if as_yuv420:
            u8 = _i420_out(u8, poses_c2w.shape[0], 2 * R, self.density_bitfield.device)
        res = super().render_clip(poses_c2w, intrinsics, H, W, *args, **kwargs)
        rgb, stats = res if want_stats else (res, None)
        T = rgb.shape[0]
        if as_uint8:
            u8 = u8 if u8 is not None else torch.empty(T, 2 * R, 2 * R, 3, device=rgb.device, dtype=torch.uint8)
            if u8.shape != (T, 2 * R, 2 * R, 3) or u8.dtype != torch.uint8 or not u8.is_contiguous():
                raise ValueError(f"out must be a contiguous uint8 [{T},{2 * R},{2 * R},3] tensor")
        native = rgb.is_cuda and self.sr_net.backend == "native"
        out = None if (as_uint8 or as_yuv420) and native else torch.empty(T, 3, 2 * R, 2 * R, device=rgb.device, dtype=torch.float32)
        with torch.autocast(rgb.device.type, enabled=False):
            if native and as_yuv420:
                # chunk by chunk as forward_native would go, so the noise planes are drawn in the same order and shapes
                for s in range(0, T, sr_frames_per_call):
                    e = min(T, s + sr_frames_per_call)
                    frames = video.frame_scratch(self, (e - s, 2 * R, 2 * R, 3))
                    self.sr_net.forward_native(rgb[s:e], noise_mode=sr_noise_mode, clamp=True, frames_per_call=sr_frames_per_call, u8_out=frames)
                    video.rgb_u8_to_i420(frames, 2 * R, 2 * R, out=u8[s:e])
            elif native:
                # libgfpp's SR kernels read the renderer's [T,N,3] frames as they are and clamp in their last epilogue
                self.sr_net.forward_native(rgb, noise_mode=sr_noise_mode, clamp=True, out=out, frames_per_call=sr_frames_per_call, u8_out=u8)
            else:
                for s in range(0, T, sr_frames_per_call):
                    e = min(T, s + sr_frames_per_call)
                    out[s:e] = self.sr_net(rgb[s:e].view(e - s, R, R, 3).permute(0, 3, 1, 2), noise_mode=sr_noise_mode).clamp(0, 1)
                    if as_uint8:
                        u8[s:e] = to_uint8(out[s:e].permute(0, 2, 3, 1))
                    elif as_yuv420:
                        video.rgb_u8_to_i420(to_uint8(out[s:e].permute(0, 2, 3, 1)).contiguous(), 2 * R, 2 * R, out=u8[s:e])
        out = u8 if as_uint8 or as_yuv420 else out
        return (out, stats) if want_stats else out


# ------------------------------------------------------------------------------------------------ torso + super-resolution
class _NativeEncoders:
    """Frequency / 2-D tiled-grid encoders through libgfpp's per-op C-ABI kernels (gfpp_freq_encode_forward,
    gfpp_grid_encode_forward): the wrapper-level API of the reference's encoders.  No CPU path."""

    def __init__(self):
        from .backend_shims import make_modules
        mods = make_modules()
        self._fr, self._ge = mods["_freqencoder"], mods["_gridencoder"]

    def freq_encode(self, x, degree):
        x = x.float().contiguous()
        B, D = x.shape
        C = D + D * 2 * degree
        out = torch.empty(B, C, dtype=torch.float32, device=x.device)
        if B:
            self._fr.freq_encode_forward(x, B, D, degree, C, out)
        return out

    def grid_encode(self, x01, embeddings, offsets, per_level_scale, base_resolution, gridtype_id, align_corners, interp_id):
        x01 = x01.float().contiguous()
        B, D = x01.shape
        Lv, C = offsets.shape[0] - 1, embeddings.shape[1]
        out = torch.empty(Lv, B, C, dtype=torch.float32, device=x01.device)
        if B:
            self._ge.grid_encode_forward(x01, embeddings.float().contiguous(), offsets, out, B, D, C, Lv, float(np.log2(per_level_scale)),
                                         base_resolution, None, gridtype_id, align_corners, interp_id)
        return out.permute(1, 0, 2).reshape(B, Lv * C)


class _TorsoGrid:
    """density_grid_torso maintenance shared by the two torso classes: update_extra_state of radnerf_torso.py:201-242 and
    radnerf_torso_sr.py:246-288 in libgfpp (gfpp.h section F).  Each class supplies `_torso_grid_condition(index, dev)` (what the
    field is conditioned on for training pose `index`), `_torso_grid_call(...)` (its C entry point) and
    `_set_torso_threshold(thr)` (writes the new mask threshold into its packed handle, no repack)."""

    def _torso_cell_noise(self, S, dev):
        """The reference's rand_like draws (radnerf_torso.py:216-227) as one [H,H,2] tensor: chunks of S cells along x, then y,
        one [chunk, 2] draw per chunk in meshgrid(x, y) order."""
        H = self.grid_size
        noise = torch.empty(H, H, 2, device=dev)
        for x0 in range(0, H, S):
            for y0 in range(0, H, S):
                nx, ny = min(S, H - x0), min(S, H - y0)
                noise[x0:x0 + nx, y0:y0 + ny] = torch.rand(nx * ny, 2, device=dev).view(nx, ny, 2)
        return noise

    def _torso_grid_ws(self, dev, need=None):
        """Device workspace of the refresh (default) or of `need` bytes (the torso query), kept across calls."""
        if need is None:
            need = _capi.lib().gfpp_torso_grid_workspace_bytes(self.grid_size)
            if need == 0:
                raise _capi.GfppError(f"the torso grid refresh does not support grid_size {self.grid_size}")
        ws = self.__dict__.get("_torso_grid_ws_buf")
        if ws is None or ws.numel() < need or ws.device != dev:
            ws = self.__dict__["_torso_grid_ws_buf"] = torch.empty(need, dtype=torch.uint8, device=dev)
        return ws

    def _torso_code_row(self, index, dev):
        """torso_individual_codes[index] as a contiguous fp32 device vector, or None without codes.  The index is checked here, on
        the host: an out-of-range row never reaches the device."""
        if self.torso_individual_embedding_dim == 0:
            return None
        n = self.torso_individual_codes.shape[0]
        if not 0 <= index < n:
            raise IndexError(f"torso code row {index} out of range for {n} torso_individual_codes")
        return self.torso_individual_codes[index].detach().to(dev, torch.float32).contiguous()

    def _require_cuda(self):
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppNoCpuPath("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        return dev

    @torch.no_grad()
    def refresh_torso_grid(self, cond, code, noise, decay=0.95, tmp_grid=None):
        """The device half of update_extra_state in libgfpp, on the current stream, no host sync: density_grid_torso (dilated
        EMA, in place).  Returns the device scalar mean_density_torso.  cond: pose6 [6] (RADNeRFTorso) or lm68 [136]
        (RADNeRFTorsowithSR); code: a row of torso_individual_codes or None; noise [H,H,2] in [0,1); tmp_grid: optional [H*H]
        fp32 tensor that receives the raw (pre-dilation) alphas at the reference's index y*H + x."""
        dev = self._require_cuda()
        H = self.grid_size
        noise = noise.to(dev, torch.float32).contiguous()
        if noise.numel() != H * H * 2:
            raise ValueError(f"noise must be [{H},{H},2]")
        g = self.density_grid_torso
        if g.dtype != torch.float32 or not g.is_contiguous():
            raise ValueError("density_grid_torso must be a contiguous fp32 buffer")
        if tmp_grid is not None and (tmp_grid.dtype != torch.float32 or not tmp_grid.is_contiguous() or tmp_grid.numel() != H * H
                                     or tmp_grid.device != dev):
            raise ValueError(f"tmp_grid must be a contiguous fp32 [{H * H}] tensor on {dev}")
        if (code is None) != (self.torso_individual_embedding_dim == 0):
            raise ValueError("code must be given iff the model has torso_individual_codes")
        if code is not None:
            code = code.to(dev, torch.float32).reshape(-1).contiguous()
        ws = self._torso_grid_ws(dev)
        mean = torch.empty(1, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            # writes density_grid_torso through its pointer: its _version does not move, so the packed handles stay valid
            self._torso_grid_call(cond, code, noise, float(decay), g.data_ptr(), mean.data_ptr(),
                                  None if tmp_grid is None else tmp_grid.data_ptr(), ws)
        self.last_launch_count = int(_capi.lib().gfpp_last_launch_count())
        return mean

    def torso_pass(self, image, weights_sum, bg_coords, poses, c, bg_color=None, lm68=None):
        """The torso part of the torso training step (radnerf_torso.py:165-193, radnerf_torso_sr.py:196-221) between frozen_head()
        and the loss, fused on libgfpp (gfpp.h section M around the training field of section H or I):

            weights_sum, image = model.frozen_head(rays_o, rays_d, cond_feat, model.individual_embeddings[idx], perturb=True, max_steps=16)
            res = model.torso_pass(image, weights_sum, bg_coords, pose6, model.torso_individual_codes[idx], bg_color=bg)        # RADNeRFTorso
            res = sr.torso_pass(image, weights_sum, bg_coords, None, sr.torso_individual_codes[idx], bg_color=bg, lm68=lm68)  # torso-SR

        image [N,3] / weights_sum [N] the head's premultiplied colour and alpha, bg_coords [...,2] with N pixels, poses the head pose
        [1,6] (convert_poses; RADNeRFTorso) or unused (RADNeRFTorsowithSR, conditioned on lm68, 136 values), c the code row
        torso_individual_codes[idx] or None without codes, bg_color None (1), one colour (3 values) or one per pixel (N x 3).
        Returns the composed recipe's flat maps: torso_alpha_map [N,1], torso_rgb_map [N,3], rgb_map [N,3] (clamped), weights_sum [N]
        and, iff some pixel is masked, deform [M,2].  The SR task reshapes rgb_map to [1,3,R,R] for its SR head, as the reference does.
        The maps are bit-identical to the composed recipe (README); gradients reach the same parameters as forward_torso's (the
        torso MLPs, the torso table, the code row, head_color_weights_encoder with torso_head_aware), deform's included.  One host
        sync (the count of masked pixels, from a pinned buffer); fp32, with autocast disabled inside; train or eval mode.  With no
        masked pixel no field runs and no output requires grad.  Inputs other than the parameters that require grad raise
        NotImplementedError, as forward_torso does."""
        dev = self._require_cuda()
        if any(torch.is_tensor(t) and t.requires_grad for t in (image, weights_sum, bg_coords, poses, lm68, bg_color)):
            raise NotImplementedError("gradients w.r.t. the head image, weights_sum, bg_coords, the pose, lm68 or bg_color are not implemented")
        dim = self.torso_individual_embedding_dim
        if (c is None) != (dim == 0) or (c is not None and (not torch.is_tensor(c) or c.numel() != dim)):
            raise ValueError(f"c must hold {dim} values (None iff the model has no torso_individual_codes)")
        field, head_aware = self._torso_pass_field(poses, None if c is None else c.to(dev), lm68, dev)
        from . import train_ops
        with torch.autocast("cuda", enabled=False):
            return train_ops.torso_pass(self, image, weights_sum, bg_coords, bg_color, field, head_aware)

    @torch.no_grad()
    def update_extra_state(self, decay=0.95, S=128, *, pose_index=None, noise=None):
        """radnerf_torso.py:201-242 / radnerf_torso_sr.py:246-288: refreshes density_grid_torso and mean_density_torso only.  The
        field is conditioned on training pose `pose_index` of `self.poses` (and `self.lm68s`), which the training task sets, with
        torso code row `pose_index` (default: random.randint, as the reference); the cell jitter comes from `noise` [H,H,2] in
        [0,1) (default: torch.rand in the reference's draw order for chunk size S).  The next render masks with the new
        min(density_thresh_torso, mean_density_torso) without a repack."""
        import random
        dev = self._require_cuda()
        if pose_index is None:
            pose_index = random.randint(0, len(self.poses) - 1)
        if not 0 <= pose_index < len(self.poses):
            raise IndexError(f"pose_index {pose_index} out of range for {len(self.poses)} training poses")
        cond = self._torso_grid_condition(pose_index, dev)
        code = self._torso_code_row(pose_index, dev)
        if noise is None:
            noise = self._torso_cell_noise(S, dev)
        mean = self.refresh_torso_grid(cond, code, noise, decay)
        self.mean_density_torso = mean.item()
        self._set_torso_threshold(float(min(self.density_thresh_torso, self.mean_density_torso)))
        # the head pack's cache key (RADNeRF._ensure_packed: head part, then (mean_density_torso, torso versions)) follows the new
        # mean without a repack: RADNeRFTorso's handle has just been given the new threshold, and RADNeRFTorsowithSR packs the head
        # field only (has_torso = 0), which the torso mean does not touch
        if self._packed is not None:
            (head_key, torso_key), packed, model, keep = self._packed
            self._packed = ((head_key, (self.mean_density_torso,) + torso_key[1:]), packed, model, keep)


class RADNeRFTorsowithSR(_TorsoGrid, RADNeRF):
    """modules/radnerfs/radnerf_torso_sr.py:17-246 (the `lm3d_radnerf_torso_sr.yaml` checkpoints; SURVEY.md 8(f) rank 3).

    Same state (`density_grid_torso`, `torso_individual_codes`, `torso_embedder.*`, `head_color_weights_encoder.*`,
    `torso_deform_net.*`, `torso_canonicial_net.*`, `sr_net.*`, blink modules) and `render(..., lm68=, eye_area_percent=,
    upscale_torso=)` result dict.  The head NeRF runs in libgfpp's fused kernels at 256x256; this variant's torso field --
    2-D position (42) + code (8) + freq-encoded jaw landmarks (126) [+ a per-pixel 4->16->32->16 encoding of the head colour and
    alpha] -> deform 64-64-2 -> tiled 2-D grid -> canonical 32-32-4 -- and the three-way composite run in libgfpp's `k_torso_sr`
    (csrc/torso_sr_kernel.cu, `torso_backend = "native"`), the SR head in libgfpp's wgmma convolution kernels (superres.py).
    `torso_backend = "torch"` keeps the first correct path -- the field as host-side PyTorch over libgfpp's per-op encoder kernels --
    as the A/B reference of the kernel; it is also what the CPU test drives with the encoders injected from the checker
    (tests/golden/torso_sr256.npz).  On the GPU both are pinned against the reference's own render() golden."""
    has_torso = False            # what gets packed for libgfpp is the head field only
    forwards_eye_area = True     # radnerf_torso_sr.py:136
    sr_input_resolution = 256
    torso_backend = "native"     # libgfpp's k_torso_sr (csrc/torso_sr_kernel.cu); "torch": the host-side field below over libgfpp's
                                 # per-op encoder kernels (the first correct path, kept as the A/B reference of the kernel)

    def __init__(self, hparams):
        super().__init__(hparams)
        hp = self.hparams
        self.register_buffer("density_grid_torso", torch.zeros(self.grid_size ** 2))
        self.mean_density_torso = 0
        self.density_thresh_torso = hp["density_thresh_torso"]
        self.torso_shrink = hp["torso_shrink"]
        self.torso_individual_embedding_dim = hp["torso_individual_embedding_dim"]
        if self.torso_individual_embedding_dim > 0:
            self.torso_individual_codes = nn.Parameter(torch.randn(hp["individual_embedding_num"], self.torso_individual_embedding_dim) * 0.1)
        self.torso_layout = GridLayout(2, log2_hashmap_size=16, desired_resolution=2048, gridtype="tiled")
        self.torso_embedder = _GridParams(self.torso_layout)
        din = (2 + 2 * 2 * 10) + (14 + 14 * 2 * 4) + self.torso_individual_embedding_dim
        self.torso_head_aware = bool(hp["torso_head_aware"])
        if self.torso_head_aware:
            self.head_color_weights_encoder = nn.Sequential(nn.Linear(4, 16), nn.LeakyReLU(0.02, True), nn.Linear(16, 32),
                                                            nn.LeakyReLU(0.02, True), nn.Linear(32, 16))
            din += 16
        self.torso_deform_net = _MLPWeights(din, 2, 64, 3)
        self.torso_canonicial_net = _MLPWeights(self.torso_layout.output_dim + din, 4, 32, 3)
        from .superres import Superresolution
        self.sr_net = Superresolution(channels=3)
        self.encoders = None      # _NativeEncoders (libgfpp per-op kernels) on first use.  Nothing in the package sets this: it is the
                                  # seam through which the CPU unit test of the host logic supplies the checker's encoders

    # ---- density_grid_torso refresh (_TorsoGrid): the field conditioned on lm68s[index], head-aware inputs zero
    def _torso_grid_condition(self, index, dev):
        return self.lm68s[index].detach().to(dev, torch.float32).reshape(136).contiguous()

    def _torso_grid_call(self, lm68, code, noise, decay, grid, mean, tmp, ws):
        lm68 = lm68.to(self.density_bitfield.device, torch.float32).reshape(-1).contiguous()
        if lm68.numel() != 136:
            raise ValueError("the torso-SR refresh takes one lm68 row of 136 values")
        st = self._torso_native_state()
        dev = self.density_bitfield.device
        _capi.check(_capi.lib().gfpp_torso_sr_grid_update(ctypes.byref(st["model"]), lm68.data_ptr(), None if code is None else code.data_ptr(),
                                                          noise.data_ptr(), decay, grid, mean, tmp, ws.data_ptr(), ws.numel(),
                                                          _capi.stream_ptr(dev)), "gfpp_torso_sr_grid_update")

    def _set_torso_threshold(self, thr):
        st = self.__dict__.get("_torso_native")
        if st is None:
            return                              # the next _torso_native_state() packs with the new threshold
        _capi.check(_capi.lib().gfpp_torso_sr_set_threshold(ctypes.byref(st["model"]), thr), "gfpp_torso_sr_set_threshold")
        st["key"] = (st["key"][0], thr, st["key"][2])   # (device, threshold, parameter pointers + versions)

    @staticmethod
    def _mlp(x, net):
        for i, lin in enumerate(net.net):
            x = F.linear(x, lin.weight)
            if i != len(net.net) - 1:
                x = F.relu(x)
        return x

    def forward_torso(self, x, poses, c=None, image=None, weights_sum=None, lm68=None):
        """radnerf_torso_sr.py:73-113 (`poses` is accepted and unused there too): x [n,2] in [-1,1], c [1,torso_code_dim] (a row of
        torso_individual_codes) or None without codes, image [n,3] / weights_sum [n,1] the head colour and alpha at the points (None:
        zeros; read only with torso_head_aware), lm68 (136 values) -> (alpha [n,1], color [n,3], dx [n,2]).
        In training mode it runs libgfpp's fused fp32 field (gfpp.h section I) and is differentiable w.r.t. the six torso MLP weights,
        the torso grid table, head_color_weights_encoder and c (with c = torso_individual_codes[index] only that row gets a gradient);
        it returns fp32 also under torch.autocast, and its values are bit-identical to the render epilogue's at the same inputs.  In
        eval mode it is the host-side field over `encoders`, without autograd."""
        if self.training:
            dev = self._require_cuda()
            if any(torch.is_tensor(t) and t.requires_grad for t in (x, image, weights_sum, lm68)):
                raise NotImplementedError("gradients w.r.t. the torso positions, the head image, weights_sum or lm68 are not implemented")
            if lm68 is None:
                raise ValueError("the torso-SR field is conditioned on lm68 (radnerf_torso_sr.py:84)")
            from . import train_ops
            to = (lambda t: None if t is None else t.to(dev))
            with torch.autocast("cuda", enabled=False):
                return train_ops.torso_sr_field(self, x.to(dev), lm68.to(dev), to(c), to(image), to(weights_sum), *train_ops.torso_sr_params(self))
        enc = self.encoders
        x = x * self.torso_shrink
        enc_x = enc.freq_encode(x, 10)
        jaw = lm68.reshape(1, 68, 2)[:, [5, 6, 7, 8, 9, 10, 11]].reshape(1, -1)
        enc_lm = enc.freq_encode(jaw.float().to(x.device), 4)
        parts = [enc_x] + ([c.reshape(1, -1).repeat(x.shape[0], 1)] if c is not None else []) + [enc_lm.repeat(x.shape[0], 1)]
        h = torch.cat(parts, dim=-1)
        if self.torso_head_aware:
            if image is None:
                image = torch.zeros(x.shape[0], 3, dtype=h.dtype, device=h.device)
                weights_sum = torch.zeros(x.shape[0], 1, dtype=h.dtype, device=h.device)
            h = torch.cat([h, self.head_color_weights_encoder(torch.cat([image, weights_sum], dim=-1))], dim=-1)
        dx = self._mlp(h, self.torso_deform_net)
        x = (x + dx).clamp(-1, 1).float()
        lay = self.torso_layout
        xf = enc.grid_encode((x + 1) / 2, self.torso_embedder.embeddings, self.torso_embedder.offsets, lay.per_level_scale,
                             lay.base_resolution, 1, False, 0)
        h = self._mlp(torch.cat([xf, h], dim=-1), self.torso_canonicial_net)
        return torch.sigmoid(h[..., :1]), torch.sigmoid(h[..., 1:]), dx

    def _torso_pass_field(self, poses, c, lm68, dev):
        """torso_pass's field: (xy, image, weights_sum) -> forward_torso's training field at the masked pixels; head-aware inputs iff
        torso_head_aware.  `poses` is unused, as in forward_torso."""
        if not torch.is_tensor(lm68) or lm68.numel() != 136:
            raise ValueError("the torso-SR field is conditioned on lm68: one frame's 68 2-D landmarks (136 values)")
        from . import train_ops
        lm, params = lm68.to(dev), train_ops.torso_sr_params(self)
        return (lambda xy, image, ws: train_ops.torso_sr_field(self, xy, lm, c, image, ws, *params)), self.torso_head_aware

    def _torso_native_state(self):
        """gfpp_torso_sr_pack once per (device, parameter versions)."""
        dev = self.density_bitfield.device
        ts = [self.density_grid_torso, self.torso_embedder.embeddings] + [l.weight for l in self.torso_deform_net.net] + \
             [l.weight for l in self.torso_canonicial_net.net]
        if self.torso_individual_embedding_dim > 0:
            ts.append(self.torso_individual_codes)
        if self.torso_head_aware:
            ts += [p for p in self.head_color_weights_encoder.parameters()]
        thr = float(min(self.density_thresh_torso, self.mean_density_torso))
        key = (dev.index, thr, tuple((t.data_ptr(), int(t._version)) for t in ts))
        st = self.__dict__.get("_torso_native")
        if st is not None and st["key"] == key:
            return st
        L = _capi.lib()
        keep = []
        d = _capi.TorsoSrDesc()
        d.torso_grid = self._grid_desc(self.torso_embedder, keep)
        for i in range(3):
            d.torso_deform_w[i] = self._w(self.torso_deform_net.net[i].weight, keep)
            d.torso_canon_w[i] = self._w(self.torso_canonicial_net.net[i].weight, keep)
        d.torso_code_dim = self.torso_individual_embedding_dim
        if self.torso_individual_embedding_dim > 0:
            d.torso_code = self._w(self.torso_individual_codes[0], keep)        # eval uses code 0 (radnerf_torso_sr.py:188)
        d.head_aware = int(self.torso_head_aware)
        if self.torso_head_aware:
            lins = [m for m in self.head_color_weights_encoder if isinstance(m, nn.Linear)]
            for i, lin in enumerate(lins):
                d.ha_w[i] = self._w(lin.weight, keep)
                d.ha_b[i] = self._w(lin.bias, keep)
        g = self.density_grid_torso
        keep.append(g)
        d.density_grid_torso = g.data_ptr()
        d.grid_size = self.grid_size
        d.density_thresh_torso = thr
        d.torso_shrink = float(self.torso_shrink)
        packed = torch.empty(L.gfpp_torso_sr_packed_bytes(), dtype=torch.uint8, device=dev)
        model = _capi.TorsoSrModel()
        with torch.cuda.device(dev):
            _capi.check(L.gfpp_torso_sr_pack(ctypes.byref(d), packed.data_ptr(), packed.numel(), ctypes.byref(model), _capi.stream_ptr(dev)),
                        "gfpp_torso_sr_pack")
        st = {"key": key, "packed": packed, "model": model, "keep": keep, "ws": None}
        self.__dict__["_torso_native"] = st
        return st

    def torso_composite_native(self, image, weights_sum, lm68, bg_coords, bg_color=None, want_maps=True, rgb_out=None):
        """Torso field + three-way composite of F frames in libgfpp (k_torso_sr): image [F,N,3] premultiplied head colour,
        weights_sum [F,N], lm68 [F,136], bg_coords [N,2], bg_color [N,3] / None (= 1).  Returns a dict of device tensors:
        rgb_map [F,N,3] (clamped) and, want_maps, torso_alpha_map [F,N], torso_rgb_map [F,N,3], deform [F,N,2], torso_pixels [F]."""
        dev = self.density_bitfield.device
        if dev.type != "cuda":
            raise _capi.GfppError("model is not on a CUDA device: libgfpp has no CPU path (call .cuda())")
        f32 = torch.float32
        st = self._torso_native_state()
        L = _capi.lib()
        image = image.to(dev, f32).contiguous()
        Fn, N = image.shape[0], image.shape[1]
        weights_sum = weights_sum.to(dev, f32).reshape(Fn, N).contiguous()
        lm68 = lm68.to(dev, f32).reshape(Fn, 136).contiguous()
        bg_coords = bg_coords.to(dev, f32).reshape(-1, 2).contiguous()
        if bg_coords.shape[0] != N:
            raise ValueError(f"bg_coords must be [{N},2] (one row per pixel)")
        fr = _capi.TorsoSrFrames()
        fr.n_frames, fr.n_rays = Fn, N
        fr.image, fr.weights_sum, fr.lm68, fr.bg_coords = image.data_ptr(), weights_sum.data_ptr(), lm68.data_ptr(), bg_coords.data_ptr()
        hold = [image, weights_sum, lm68, bg_coords]
        if bg_color is not None:
            if not torch.is_tensor(bg_color):
                bg_color = torch.full((N, 3), float(bg_color), device=dev, dtype=f32)
            bg_color = bg_color.to(dev, f32).reshape(-1, 3)
            if bg_color.shape[0] == 1:
                bg_color = bg_color.expand(N, 3)
            elif bg_color.shape[0] != N:
                raise ValueError(f"bg_color must have 1 or {N} rows, got {bg_color.shape[0]}")
            bg_color = bg_color.contiguous()
            fr.bg_color = bg_color.data_ptr()
            hold.append(bg_color)
        res = {"rgb_map": rgb_out if rgb_out is not None else torch.empty(Fn, N, 3, device=dev, dtype=f32)}
        if res["rgb_map"].dtype != f32 or not res["rgb_map"].is_contiguous() or res["rgb_map"].numel() != Fn * N * 3:
            raise ValueError(f"rgb_out must be a contiguous fp32 [{Fn},{N},3] tensor")
        ptrs = [None] * 4
        if want_maps:
            res["torso_alpha_map"] = torch.empty(Fn, N, device=dev, dtype=f32)
            res["torso_rgb_map"] = torch.empty(Fn, N, 3, device=dev, dtype=f32)
            res["deform"] = torch.empty(Fn, N, 2, device=dev, dtype=f32)
            res["torso_pixels"] = torch.empty(Fn, device=dev, dtype=torch.int32)
            ptrs = [res[k].data_ptr() for k in ("torso_alpha_map", "torso_rgb_map", "deform", "torso_pixels")]
        need = L.gfpp_torso_sr_workspace_bytes(Fn)
        if st["ws"] is None or st["ws"].numel() < need:
            st["ws"] = torch.empty(need, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _capi.check(L.gfpp_torso_sr_composite(ctypes.byref(st["model"]), ctypes.byref(fr), res["rgb_map"].data_ptr(), *ptrs,
                                                  st["ws"].data_ptr(), st["ws"].numel(), _capi.stream_ptr(dev)), "gfpp_torso_sr_composite")
        del hold
        return res

    def _head(self, rays_o, rays_d, cond_feat, dt_gamma, max_steps, T_thresh, noise=None):
        """Premultiplied head colour, alpha and normalised depth of one frame from libgfpp (background 0 => rgb_map == image).
        noise: optional [N] jittered ray starts (render_frames)."""
        N = rays_o.numel() // 3
        res = self.render_frames(cond_feat.reshape(1, -1), rays_o=rays_o.reshape(1, -1, 3), rays_d=rays_d.reshape(1, -1, 3),
                                 bg_color=torch.zeros(N, 3, device=self.density_bitfield.device), dt_gamma=dt_gamma,
                                 max_steps=max_steps, T_thresh=T_thresh, noise=noise)
        return res["rgb_map"].view(N, 3), res["weights_sum"].view(N), res["depth_map"].view(N)

    @torch.no_grad()
    def render(self, rays_o, rays_d, cond, bg_coords, poses, index=0, dt_gamma=0, bg_color=None, perturb=False, force_all_rays=False,
               max_steps=1024, T_thresh=1e-4, upscale_torso=False, lm68=None, eye_area_percent=None, **kwargs):
        if self.training:
            raise NotImplementedError(f"{type(self).__name__} renders for inference only; training covers the head field (RADNeRF)")
        if lm68 is None:
            raise ValueError("the torso-SR field is conditioned on lm68 (radnerf_torso_sr.py:84)")
        R = self.sr_input_resolution
        prefix = rays_o.shape[:-1]
        N = rays_o.numel() // 3
        if N != R * R:
            raise ValueError(f"SR models render the NeRF at {R}x{R} (radnerf_torso_sr.py:229)")
        if self.encoders is None:
            self.encoders = _NativeEncoders()
        dev = self.density_bitfield.device
        with torch.autocast(dev.type, enabled=False):
            cond_feat = self.cal_cond_feat(cond.to(dev), eye_area_percent=eye_area_percent)
            # perturb: the marching draw comes first, the SR head's noise planes after it (radnerf_torso_sr.py:166-181 marches first)
            jitter = {"noise": self._ray_start_noise(N)} if perturb else {}
            image, weights_sum, depth = self._head(rays_o.to(dev), rays_d.to(dev), cond_feat, dt_gamma, max_steps, T_thresh, **jitter)
            bg_coords = bg_coords.to(dev).contiguous().view(-1, 2)
            bg = 1 if bg_color is None else (bg_color.to(dev).reshape(-1, 3) if torch.is_tensor(bg_color) else bg_color)
            code = self.torso_individual_codes[0] if self.torso_individual_embedding_dim > 0 else None
            G = self.grid_size
            occ = F.grid_sample(self.density_grid_torso.view(1, 1, G, G), bg_coords.view(1, -1, 1, 2), align_corners=True).view(-1)
            mask = occ > min(self.density_thresh_torso, self.mean_density_torso)
            results = {}
            noise_mode = kwargs.get("sr_noise_mode", "random")
            if self.torso_backend == "native":
                tr = self.torso_composite_native(image.view(1, N, 3), weights_sum.view(1, N), lm68.reshape(1, 136), bg_coords,
                                                 None if not torch.is_tensor(bg) and bg == 1 else bg)
                if bool(mask.any()):
                    results["deform"] = tr["deform"][0][mask]
                rgb_image = tr["rgb_map"].view(1, R, R, 3).permute(0, 3, 1, 2)
                torso_bg = tr["torso_rgb_map"].view(1, R, R, 3).permute(0, 3, 1, 2)
                results.update({"torso_alpha_map": tr["torso_alpha_map"].view(N, 1), "torso_rgb_map": torso_bg, "depth_map": depth.view(*prefix),
                                "rgb_map": rgb_image, "sr_rgb_map": self.sr_net(rgb_image, noise_mode=noise_mode).clamp(0, 1)})
                if upscale_torso:
                    results["sr_torso_rgb_map"] = self.sr_net(torso_bg, noise_mode=noise_mode).clamp(0, 1)
                return results
            torso_alpha = torch.zeros(N, 1, device=dev)
            torso_color = torch.zeros(N, 3, device=dev)
            if bool(mask.any()):
                a, c, deform = self.forward_torso(bg_coords[mask], poses, code, image[mask] if self.torso_head_aware else None,
                                                  weights_sum.unsqueeze(-1)[mask] if self.torso_head_aware else None, lm68=lm68)
                torso_alpha[mask] = a.float()
                torso_color[mask] = c.float()
                results["deform"] = deform
            torso_bg = torso_color * torso_alpha + bg * (1 - torso_alpha)
            img = (image + (1 - weights_sum).unsqueeze(-1) * torso_bg).clamp(0, 1)
            rgb_image = img.reshape(1, R, R, 3).permute(0, 3, 1, 2)
            torso_bg = torso_bg.reshape(1, R, R, 3).permute(0, 3, 1, 2)
            results.update({"torso_alpha_map": torso_alpha, "torso_rgb_map": torso_bg, "depth_map": depth.view(*prefix),
                            "rgb_map": rgb_image, "sr_rgb_map": self.sr_net(rgb_image, noise_mode=noise_mode).clamp(0, 1)})
            if upscale_torso:
                results["sr_torso_rgb_map"] = self.sr_net(torso_bg, noise_mode=noise_mode).clamp(0, 1)
        return results

    @torch.no_grad()
    def render_clip(self, poses_c2w, intrinsics, H=256, W=256, cond_seq=None, bg_color=None, bg_coords=None, lm68_seq=None,
                    eye_area_percent=None, dt_gamma=None, max_steps=None, T_thresh=1e-2, sr_noise_mode="random", cond_feat=None,
                    as_uint8=False, as_rgba=False, as_yuv420=False, **unused):
        """Clip API of the torso-SR model -> the clamped 512x512 frames [T,3,512,512].  With the native backends (the default) every
        stage runs in libgfpp chunk by chunk -- head field with rays generated in-kernel, torso-SR field + composite, SR head -- with
        no per-frame host work; with a "torch" backend it falls back to frame-by-frame `render()`.  poses_c2w [T,4,4] (c2w,
        dataset.poses), cond_seq [T,1,C] (or cond_feat [T,64] precomputed), lm68_seq [T,136], eye_area_percent [T] or None.
        as_uint8: returns the video frames uint8 [T,512,512,3] (HWC) `(rgb*255).int()` instead, written by the SR head's last kernel
        chunk by chunk into `out` (optional preallocated buffer of that shape); no fp32 512x512 frame is written then.
        as_yuv420: the same frames as planar I420, uint8 [T,512*512*3/2] (video.rgb_u8_to_i420), each chunk's uint8 frames
        converted from a scratch buffer the model keeps into `out`; the noise planes are drawn as with as_uint8.
        as_rgba raises ValueError (_no_sr_matte), and so does as_yuv420 with as_uint8."""
        _no_sr_matte(as_rgba)
        if as_yuv420 and as_uint8:
            raise ValueError("as_yuv420 is a frame format of its own: it cannot be combined with as_uint8 or as_rgba")
        from .dist import to_uint8
        from .scene import cond_window, convert_poses, get_rays
        R = self.sr_input_resolution
        if (H, W) != (R, R):
            raise ValueError(f"SR models render the NeRF at {R}x{R} (radnerf_torso_sr.py:229)")
        hp = self.hparams
        T = poses_c2w.shape[0]
        dev = self.density_bitfield.device
        native = self.torso_backend == "native" and self.sr_net.backend == "native"
        u8 = None
        if as_uint8:
            u8 = unused.get("out")
            u8 = u8 if u8 is not None else torch.empty(T, 2 * R, 2 * R, 3, device=dev, dtype=torch.uint8)
            if u8.shape != (T, 2 * R, 2 * R, 3) or u8.dtype != torch.uint8 or not u8.is_contiguous():
                raise ValueError(f"out must be a contiguous uint8 [{T},{2 * R},{2 * R},3] tensor")
        yuv = _i420_out(unused.get("out"), T, 2 * R, dev) if as_yuv420 else None
        out = None if (as_uint8 or as_yuv420) and native else torch.empty(T, 3, 2 * R, 2 * R, device=dev, dtype=torch.float32)
        if native:
            # everything in libgfpp, chunk by chunk: head field (rays generated in-kernel, background 0 => premultiplied colour),
            # torso-SR field + composite, SR head; no per-frame host work
            fpc = min(8, int(unused.get("frames_per_call", 8)))     # the SR workspace is 68 MB per frame
            if cond_feat is None:                                   # [T,64] precomputed (sharded clips: dist.render_clip_sharded) or from the sequence
                cond_feat = self.cal_cond_feat_clip(cond_seq.to(dev), eye_area_percent=eye_area_percent)
            poses_c2w = poses_c2w.to(dev, torch.float32)
            zero_bg = torch.zeros(R * R, 3, device=dev)
            with torch.autocast(dev.type, enabled=False):
                for s in range(0, T, fpc):
                    e = min(T, s + fpc)
                    hd = self.render_frames(cond_feat[s:e], poses_c2w=poses_c2w[s:e], intrinsics=intrinsics, H=H, W=W, bg_color=zero_bg,
                                            dt_gamma=hp["dt_gamma"] if dt_gamma is None else dt_gamma,
                                            max_steps=hp["max_steps"] if max_steps is None else max_steps, T_thresh=T_thresh)
                    tr = self.torso_composite_native(hd["rgb_map"], hd["weights_sum"], lm68_seq[s:e].reshape(e - s, 136), bg_coords, bg_color,
                                                     want_maps=False)
                    frames = video.frame_scratch(self, (e - s, 2 * R, 2 * R, 3)) if as_yuv420 else None if u8 is None else u8[s:e]
                    self.sr_net.forward_native(tr["rgb_map"], noise_mode=sr_noise_mode, clamp=True, out=None if out is None else out[s:e],
                                               frames_per_call=fpc, u8_out=frames)
                    if as_yuv420:
                        video.rgb_u8_to_i420(frames, 2 * R, 2 * R, out=yuv[s:e])
            return yuv if as_yuv420 else u8 if as_uint8 else out
        if cond_seq is None:
            raise ValueError("the frame-by-frame host path of the torso-SR clip needs cond_seq (cond_feat is only taken by the all-native path)")
        for t in range(T):
            rays_o, rays_d = get_rays(poses_c2w[t].cpu(), intrinsics, H, W)
            res = self.render(rays_o.to(dev), rays_d.to(dev), cond_window(cond_seq, t, self.smo_win_size).to(dev), bg_coords,
                              convert_poses(poses_c2w[t].cpu().view(1, 4, 4)).to(dev), index=t,
                              dt_gamma=hp["dt_gamma"] if dt_gamma is None else dt_gamma, bg_color=bg_color,
                              max_steps=hp["max_steps"] if max_steps is None else max_steps, T_thresh=T_thresh, lm68=lm68_seq[t].reshape(1, -1),
                              eye_area_percent=None if eye_area_percent is None else eye_area_percent[t].reshape(1, 1),
                              sr_noise_mode=sr_noise_mode)
            out[t] = res["sr_rgb_map"][0]
            if as_uint8:
                u8[t] = to_uint8(out[t].permute(1, 2, 0))
            elif as_yuv420:
                video.rgb_u8_to_i420(to_uint8(out[t].permute(1, 2, 0)).contiguous(), 2 * R, 2 * R, out=yuv[t:t + 1])
        return yuv if as_yuv420 else u8 if as_uint8 else out


# ------------------------------------------------------------------------------------------------ torso model
class RADNeRFTorso(_TorsoGrid, RADNeRF):
    has_torso = True
    trains_field = False
    forwards_eye_area = False

    def __init__(self, hparams):
        super().__init__(hparams)
        hp = self.hparams
        if hp.get("torso_head_aware", False):
            raise NotImplementedError("torso_head_aware belongs to the SR configs (SURVEY.md 8(f) rank 3)")
        # radnerf_torso.py:18-49
        self.register_buffer("density_grid_torso", torch.zeros([self.grid_size ** 2]))
        self.mean_density_torso = 0
        self.density_thresh_torso = hp["density_thresh_torso"]
        self.torso_shrink = hp["torso_shrink"]
        self.torso_individual_embedding_num = hp["individual_embedding_num"]
        self.torso_individual_embedding_dim = hp["torso_individual_embedding_dim"]
        if self.torso_individual_embedding_dim > 0:
            self.torso_individual_codes = nn.Parameter(torch.randn(self.torso_individual_embedding_num, self.torso_individual_embedding_dim) * 0.1)
        self.torso_embedder = _GridParams(GridLayout(2, log2_hashmap_size=16, desired_resolution=2048, gridtype="tiled"))
        din = (2 + 2 * 2 * 10) + (6 + 6 * 2 * 4) + self.torso_individual_embedding_dim
        self.torso_deform_net = _MLPWeights(din, 2, 64, 3)
        self.torso_canonicial_net = _MLPWeights(32 + din, 4, 32, 3)

    def _fill_desc(self, d, keep):
        super()._fill_desc(d, keep)
        d.has_torso = 1
        d.torso_grid = self._grid_desc(self.torso_embedder, keep)
        for i in range(3):
            d.torso_deform_w[i] = self._w(self.torso_deform_net.net[i].weight, keep)
            d.torso_canon_w[i] = self._w(self.torso_canonicial_net.net[i].weight, keep)
        d.torso_code_dim = self.torso_individual_embedding_dim
        if self.torso_individual_embedding_dim > 0:
            d.torso_code = self._w(self.torso_individual_codes[0], keep)  # radnerf_torso.py:160-162
        g = self.density_grid_torso
        keep.append(g)
        d.density_grid_torso = g.data_ptr()
        # mean_density_torso is a plain attribute that is NOT in the checkpoint (=> 0 after load, radnerf_torso.py:22,167)
        d.density_thresh_torso = float(min(self.density_thresh_torso, self.mean_density_torso))
        d.torso_shrink = float(self.torso_shrink)

    def _torso_pack_sources(self):
        # density_grid_torso is read in place through its pointer (the refresh writes it there): not a packed copy
        ts = [self.torso_embedder.embeddings] + [l.weight for l in self.torso_deform_net.net] + [l.weight for l in self.torso_canonicial_net.net]
        if self.torso_individual_embedding_dim > 0:
            ts.append(self.torso_individual_codes)
        return ts

    def forward_torso(self, x, poses, c=None):
        """radnerf_torso.py:51-84 in libgfpp (fp32): x [n,2] in [-1,1], poses [1,6] (convert_poses of the head pose), c
        [1,torso_code_dim] (a row of torso_individual_codes) or None without codes -> (alpha [n,1], color [n,3], dx [n,2]).
        In training mode it is differentiable w.r.t. the six torso MLP weights, the torso grid table and c (gfpp.h section H: fused
        fp32 forward and backward reading the parameters in place; with c = torso_individual_codes[index] only that row gets a
        gradient), and returns fp32 also under torch.autocast; its values are bit-identical to the eval-mode query's.  In eval mode
        it is the packed model's query (k_torso_query), without autograd."""
        dev = self._require_cuda()
        if self.training:
            if (torch.is_tensor(x) and x.requires_grad) or (torch.is_tensor(poses) and poses.requires_grad):
                raise NotImplementedError("gradients w.r.t. the torso positions or the head pose are not implemented")
            from . import train_ops
            with torch.autocast("cuda", enabled=False):
                return train_ops.torso_field(self, x.to(dev), poses.to(dev), None if c is None else c.to(dev), *self._torso_field_params())
        with torch.no_grad():
            return self._forward_torso_eval(x, poses, c, dev)

    def _torso_field_params(self):
        """The parameters train_ops.torso_field takes: the six torso MLP weights, then the torso grid table."""
        return ([self.torso_deform_net.net[i].weight for i in range(3)] + [self.torso_canonicial_net.net[i].weight for i in range(3)] +
                [self.torso_embedder.embeddings])

    def _torso_pass_field(self, poses, c, lm68, dev):
        """torso_pass's field: (xy, image, weights_sum) -> forward_torso's training field at the masked pixels (no head-aware inputs)."""
        if not torch.is_tensor(poses) or poses.numel() != 6:
            raise ValueError("RADNeRFTorso.torso_pass takes one head pose [1,6] (convert_poses)")
        from . import train_ops
        p6, params = poses.to(dev), self._torso_field_params()
        return (lambda xy, image, ws: train_ops.torso_field(self, xy, p6, c, *params)), False

    def _forward_torso_eval(self, x, poses, c, dev):
        _, _, model, _ = self._ensure_packed()
        f32 = torch.float32
        xy = x.to(dev, f32).reshape(-1, 2).contiguous()
        pose6 = poses.to(dev, f32).reshape(-1).contiguous()
        if pose6.numel() != 6:
            raise ValueError("forward_torso takes one pose [1,6] (convert_poses)")
        if (c is None) != (self.torso_individual_embedding_dim == 0):
            raise ValueError("c must be given iff the model has torso_individual_codes")
        code = None if c is None else c.to(dev, f32).reshape(-1).contiguous()
        n = xy.shape[0]
        alpha, color, dx = (torch.empty(n, k, device=dev, dtype=f32) for k in (1, 3, 2))
        ws = self._torso_grid_ws(dev, _capi.lib().gfpp_torso_query_workspace_bytes())
        with torch.cuda.device(dev):
            _capi.check(_capi.lib().gfpp_torso_query(ctypes.byref(model), xy.data_ptr(), n, pose6.data_ptr(),
                                                     None if code is None else code.data_ptr(), alpha.data_ptr(), color.data_ptr(),
                                                     dx.data_ptr(), ws.data_ptr(), ws.numel(), _capi.stream_ptr(dev)), "gfpp_torso_query")
        return alpha, color, dx

    # ---- density_grid_torso refresh (_TorsoGrid): the field conditioned on convert_poses(poses[index])
    def _torso_grid_condition(self, index, dev):
        from .scene import convert_poses
        return convert_poses(self.poses[index].detach().cpu().float().reshape(1, 4, 4)).to(dev).reshape(6)

    def _torso_grid_call(self, pose6, code, noise, decay, grid, mean, tmp, ws):
        _, _, model, _ = self._ensure_packed()
        dev = self.density_bitfield.device
        pose6 = pose6.to(dev, torch.float32).reshape(-1).contiguous()
        if pose6.numel() != 6:
            raise ValueError("the torso refresh takes one pose6 of 6 values (convert_poses)")
        _capi.check(_capi.lib().gfpp_torso_grid_update(ctypes.byref(model), pose6.data_ptr(), None if code is None else code.data_ptr(),
                                                       noise.data_ptr(), decay, grid, mean, tmp, ws.data_ptr(), ws.numel(),
                                                       _capi.stream_ptr(dev)), "gfpp_torso_grid_update")

    def _set_torso_threshold(self, thr):
        if self._packed is None:
            return                              # the next _ensure_packed() packs with the new mean_density_torso
        _capi.check(_capi.lib().gfpp_model_set_torso_threshold(ctypes.byref(self._packed[2]), thr), "gfpp_model_set_torso_threshold")

    def torso_mask(self, bg_coords):
        """radnerf_torso.py:166-169 (host-side helper used only to shape the `deform` result like the reference)."""
        G = self.grid_size
        thr = min(self.density_thresh_torso, self.mean_density_torso)
        occ = F.grid_sample(self.density_grid_torso.view(1, 1, G, G), bg_coords.to(self.density_grid_torso.device).float().view(1, -1, 1, 2), align_corners=True).view(-1)
        return occ > thr
