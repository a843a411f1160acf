"""Reference-side integration: SceneDreamer's `Generator` on the fused H100 kernels, with ZERO edits to the reference.

How the hook gets in.  The reference's `imaginaire/generators/scenedreamer.py:13` imports the `voxlib` extension by name;
with `dropin/` on PYTHONPATH that is `dropin/voxlib.py`, which calls `install_import_hook()` below.  The hook waits for
`imaginaire.generators.scenedreamer` to finish importing and then patches the `Generator` CLASS (`install`), so every
instance -- however it is wrapped (`WrappedModel`, DDP, `ModelAverage.averaged_model`, `utils/trainer.py:192-202`) --
runs the fused path; `inference.py` and `train.py` stay untouched.  `SDB200_FUSED=0` in the environment keeps the
reference's own composition (which, with dropin/ on the path, still runs on this library's DDA / PE / hash-grid kernels).

What is replaced.
  * `Generator._forward_perpix` (scenedreamer.py:313-428), the body of the per-pixel path.  Without autograd
    (`inference_givenstyle*`, `dis_forward` of trainers/gancraft.py:215-217): `sdb_sky_forward` + `sdb_render_rays_forward`.
    Under autograd (`gen_update`): the recording forward + fused backward (render.render_rays_train); gradients land on
    the module's own Parameters (hash_encoder.embeddings, render_net.*, sky_net.*) and on the incoming z / global_enc.
  * The tile loop of `inference_givenstyle*` (scenedreamer.py:600-628) is left in place but does no per-tile render any
    more: the tiles it cuts are VIEWS of the frame-sized tensors `voxlib.ray_voxel_intersection_perspective` returned, so
    the first tile of a frame triggers ONE fused launch over the whole padded frame (`_FrameCache`) and every tile --
    this one included -- gets its window of that result (per-pixel features do not depend on tile boundaries:
    deterministic sampling, frame-global `sky_avg`; DESIGN.md section 1, "Tiling equivalence").  No redundant rays, one
    launch per frame.

Cache validity (the weights may change between calls in ways torch's version counter does not see -- `param.data.copy_()`
in utils/model_average.py): every public entry of the generator (`forward`, `inference_givenstyle*`) starts a new
*epoch*; packed weights, pre-blended table and frame results never outlive the epoch they were built in, and inside an
epoch they are additionally keyed on tensor identity (a held reference, not an address) and `_version`.

The returned 12-tuple keeps the reference's order (scenedreamer.py:427-428).  Callers in the reference use only
`net_out` (0) and, in the depth variant, `weights` (2) and `rand_depth` (4) (scenedreamer.py:462-467, :618-621,
:812-816); per-sample network outputs the fused kernel never materialises (net_out_s, net_out_c, ...) are None.
"""
import functools
import importlib.abc
import importlib.util
import os
import sys

import torch

from . import optim, render, rendercnn, worldgen

TARGET_MODULE = 'imaginaire.generators.scenedreamer'
PUBLIC_ENTRIES = ('forward', 'inference_givenstyle', 'inference_givenstyle_depth')
DEFAULT_PRECISION = render.PRECISION_FP16X3


def enabled():
    return os.environ.get('SDB200_FUSED', '1') not in ('0', 'false', 'False', 'off')


# ------------------------------------------------------------------------------------------------
# per-instance state
# ------------------------------------------------------------------------------------------------
class _FrameCache:
    """Result of ONE fused launch over the padded frame the current tiles are windows of."""

    def __init__(self):
        self.clear()

    def clear(self):
        self.key, self.held, self.out = None, None, None

    def lookup(self, key_tensors, epoch, extra):
        key = (epoch, extra) + tuple((id(t), t._version) for t in key_tensors)
        if self.key == key and all(a is b for a, b in zip(self.held, key_tensors)):
            return self.out, key
        return None, key

    def store(self, key, key_tensors, out):
        self.key, self.held, self.out = key, list(key_tensors), out


class _FusedState:
    def __init__(self, gen, precision):
        self._gen_label_trans = lambda: gen.label_trans
        self._lut = None
        self.precision = precision
        self.epoch = 0
        self.renderer, self.renderer_key, self.renderer_epoch, self.cnn_epoch = None, None, -1, -1
        self.cnn, self.cnn_key, self.cnn_precision = None, None, rendercnn.PRECISION_FP16X3
        self.frame = _FrameCache()
        self.stats = {'fused_calls': 0, 'frame_launches': 0, 'tile_hits': 0, 'train_calls': 0, 'reference_calls': 0,
                      'cnn_frame_launches': 0, 'cnn_tile_hits': 0, 'cnn_calls': 0, 'cnn_reference_calls': 0}

    @property
    def lut(self):
        """mc id -> reduced label with ignore -> dirt folded in (mc_utils.py:241-246), built on first use."""
        if self._lut is None:
            lt = self._gen_label_trans()
            self._lut = render.reduced_label_lut(lt.mcid2rdid_lut, lt.ignore_id, lt.dirt_id)
        return self._lut

    def new_epoch(self):
        self.epoch += 1
        self.frame.clear()
        if self.renderer is not None:
            self.renderer.invalidate()
        self.cnn, self.cnn_key = None, None

    def get_cnn(self, gen):
        """Tensor-core RenderCNN engine over the generator's own `denoiser.*` tensors, or None if the module is not
        SceneDreamer's RenderCNN (64 -> 256 -> 3)."""
        if self.cnn_epoch == self.epoch and self.cnn_key is not None:
            return self.cnn
        self.cnn_epoch = self.epoch
        den = getattr(gen, 'denoiser', None)
        if den is None:
            return None
        P = {'denoiser.' + k: v for k, v in den.state_dict().items()}
        key = (self.epoch, tuple((k, v.data_ptr(), v._version) for k, v in P.items()))
        if self.cnn_key != key:
            self.cnn = rendercnn.RenderCNNEngine(P, self.cnn_precision) if rendercnn.supported(P) else None
            self.cnn_key = key
        return self.cnn

    def get_renderer(self, gen):
        # inside an epoch (one public call of the generator) the weights cannot change behind torch's back: the state-dict scan
        # below is done once per epoch, not once per tile of the reference's tile loop (40 scans x ~0.3 ms per frame)
        if self.renderer is not None and self.renderer_epoch == self.epoch and not torch.is_grad_enabled():
            return self.renderer
        self.renderer_epoch = self.epoch
        mods = (('render_net', gen.render_net), ('sky_net', gen.sky_net), ('hash_encoder', gen.hash_encoder))
        P = {}
        for prefix, mod in mods:
            for k, v in mod.state_dict().items():
                P[prefix + '.' + k] = v
        dims = tuple(gen.voxel.voxel_t.shape)
        # state_dict() hands out detached aliases: identity is the storage, _version is shared with the Parameter
        key = (self.epoch, dims, tuple((k, v.data_ptr(), v._version) for k, v in P.items()))
        if self.renderer_key != key:
            he = gen.hash_encoder
            self.renderer = render.FusedPerPixelRenderer(
                P, dims, self.lut, he.per_level_scale, precision=self.precision, preblend=True,
                base_res=he.base_resolution, log2_T=he.log2_hashmap_size, L=he.num_levels)
            self.renderer_key = key
        return self.renderer


def _state(gen):
    st = gen.__dict__.get('_sdb200')
    if st is None:
        st = _FusedState(gen, getattr(type(gen), '_sdb200_precision', DEFAULT_PRECISION))
        gen.__dict__['_sdb200'] = st
    return st


def _live_params(gen):
    """Parameters (not detached) under the reference's state-dict names, for the autograd path."""
    if os.environ.get('SDB200_ADAM', '1') != '0':
        emb = getattr(gen.hash_encoder, 'embeddings', None)
        if emb is not None and not getattr(emb, '_sdb200_table', False):
            optim.tag_table(emb)                                # its Adam step is taken over by the one-pass kernel (optim.py)
    P = {}
    for prefix, mod in (('render_net', gen.render_net), ('sky_net', gen.sky_net), ('hash_encoder', gen.hash_encoder)):
        for k, v in mod.named_parameters():
            P[prefix + '.' + k] = v
        for k, v in mod.named_buffers():
            P.setdefault(prefix + '.' + k, v)
    return P


# ------------------------------------------------------------------------------------------------
# which configurations the fused kernels cover (everything else keeps the reference's composition)
# ------------------------------------------------------------------------------------------------
def supported(gen, voxel_id, z, global_enc):
    """The fused path covers what both SceneDreamer configs use (configs/scenedreamer_{train,inference}.yaml):
    no view-direction input to the MLP, segmentation labels on, clipped feature blending, global sky average, AMP off (under
    autocast the reference composition runs instead, over the drop-in ops -- the grid encoder then takes its float16 table path)."""
    rn = gen.render_net
    return bool(
        not torch.is_autocast_enabled() and
        z is not None and global_enc is not None and voxel_id.is_cuda and
        gen.clip_feat_map is True and gen.keep_sky_out and gen.keep_sky_out_avgpool and gen.sky_global_avgpool and
        not gen.sample_use_box_boundaries and gen.raw_noise_std == 0 and
        gen.pe_params[2] == 0 and gen.pe_params[3] is False and          # raydirs_in is None (scenedreamer.py:331)
        getattr(rn, 'fc_viewdir', None) is None and getattr(rn, 'use_seg', True) and
        gen.pe_params_sky[0] == 5 and bool(gen.pe_params_sky[1]) and
        getattr(gen.hash_encoder, 'input_dim', 5) == 5 and getattr(gen.hash_encoder, 'level_dim', 8) == 8 and
        getattr(gen.hash_encoder, 'gridtype', 'hash') == 'hash' and not getattr(gen.hash_encoder, 'align_corners', False) and
        global_enc.shape[-1] == 2)


def _needs_grad(gen, z, global_enc):
    if not torch.is_grad_enabled():
        return False
    if z.requires_grad or global_enc.requires_grad:
        return True
    for mod in (gen.render_net, gen.hash_encoder, gen.sky_net):
        if any(q.requires_grad for q in mod.parameters()):
            return True
    return False


# ------------------------------------------------------------------------------------------------
# frame detection: is this call a window of a frame-sized raycast result?
# ------------------------------------------------------------------------------------------------
def _window_of(t, base_shape_tail, lead):
    """If `t` ([1, (2,) h, w, ...]) is a window of a contiguous base tensor [(2,) HB, WB, *tail] return
    (base, h0, w0, HB, WB), else None.  `lead` = number of leading dims of the base before H (0 or 1)."""
    base = t._base
    if base is None or t.shape[0] != 1 or base.dim() != lead + 2 + len(base_shape_tail) or not base.is_contiguous():
        return None
    if tuple(base.shape[lead + 2:]) != tuple(base_shape_tail):
        return None
    HB, WB = int(base.shape[lead]), int(base.shape[lead + 1])
    inner = 1
    for v in base_shape_tail:
        inner *= int(v)
    v = t[0]                                                 # [(2,) h, w, *tail]
    want = ((HB * WB * inner,) if lead else ()) + (WB * inner, inner) + tuple(base.stride()[lead + 2:])
    if tuple(v.stride()) != want or (lead and v.shape[0] != base.shape[0]):
        return None
    off = t.storage_offset() - base.storage_offset()
    if off < 0:
        return None
    h0, rem = divmod(off, WB * inner)
    w0, rem = divmod(rem, inner)
    h, w = int(v.shape[lead]), int(v.shape[lead + 1])
    if rem != 0 or h0 + h > HB or w0 + w > WB:
        return None
    return base, h0, w0, HB, WB


def _frame_window(voxel_id, depth2, raydirs):
    """-> (bases, h0, w0, h, w) when the three tensors are the SAME window of one frame, else None."""
    M = voxel_id.shape[3]
    a = _window_of(voxel_id, (M, 1), 0)
    b = _window_of(depth2, (M, 1), 1)
    c = _window_of(raydirs, (1, 3), 0)
    if a is None or b is None or c is None:
        return None
    if a[1:] != b[1:] or a[1:] != c[1:]:
        return None
    h, w = int(voxel_id.shape[1]), int(voxel_id.shape[2])
    if h == a[3] and w == a[4]:
        return None                                          # the whole frame in one call: nothing to cache
    return (a[0], b[0], c[0]), a[1], a[2], h, w


def _tuple12(out, sky_mask, sky_only_mask):
    total = out['total_weight'].unsqueeze(-1).unsqueeze(-1)
    return (out['net_out'], None, out['weights'], total, out['rand_depth'], None, None, out['sky'].unsqueeze(-2), None,
            sky_mask, sky_only_mask, None)


# ------------------------------------------------------------------------------------------------
# the replacement body
# ------------------------------------------------------------------------------------------------
def fused_forward_perpix(self, blk_feats, voxel_id, depth2, raydirs, cam_ori_t, z, global_enc):
    """Replacement body of Generator._forward_perpix (same arguments, same return order)."""
    st = _state(self)
    reference = type(self)._sdb200_reference_forward_perpix
    if not enabled() or not supported(self, voxel_id, z, global_enc):
        st.stats['reference_calls'] += 1
        return reference(self, blk_feats, voxel_id, depth2, raydirs, cam_ori_t, z, global_enc)
    needs_grad = _needs_grad(self, z, global_enc)
    N, H, W = voxel_id.shape[:3]
    if needs_grad:
        # differentiating through a caller-supplied sky_avg or through views of different scenes is left to the reference
        one_scene = global_enc.shape[0] == 1 or bool((global_enc == global_enc[:1]).all())
        if hasattr(self, 'sky_avg') or not one_scene:
            st.stats['reference_calls'] += 1
            return reference(self, blk_feats, voxel_id, depth2, raydirs, cam_ori_t, z, global_enc)
    uniforms = None
    if not self.coarse_deterministic_sampling:
        uniforms = torch.rand(N, H, W, self.num_samples + 1, 1, dtype=torch.float32, device=voxel_id.device)
    sky_mask = voxel_id[:, :, :, [-1], :] == 0
    sky_only_mask = voxel_id[:, :, :, [0], :] == 0
    kw = dict(num_samples=self.num_samples, sample_depth=self.sample_depth, dists_scale=self.dists_scale)
    if needs_grad:
        # one recorded pass per view (one style code each); the frame mean of the sky features is per view as well
        # (scenedreamer.py:395 averages over dims 1,2 only), so a batch is exactly the concatenation of its views
        st.stats['train_calls'] += 1
        he = self.hash_encoder
        P = _live_params(self)
        outs = []
        for i in range(N):
            outs.append(render.render_rays_train(
                P, voxel_id[i:i + 1].contiguous(), depth2[i:i + 1].contiguous(), raydirs[i:i + 1].contiguous(),
                cam_ori_t[i:i + 1], z[i:i + 1], global_enc[:1], [float(v) for v in self.voxel.voxel_t.shape], st.lut,
                he.per_level_scale, uniforms=None if uniforms is None else uniforms[i:i + 1],
                base_res=he.base_resolution, log2_T=he.log2_hashmap_size, L=he.num_levels, **kw))
        out = {k: torch.cat([o[k] for o in outs], 0) for k in ('net_out', 'total_weight', 'weights', 'rand_depth', 'sky')}
        return _tuple12(out, sky_mask, sky_only_mask)
    st.stats['fused_calls'] += 1
    r = st.get_renderer(self)
    sky_attr = getattr(self, 'sky_avg', None)                  # set once per frame by inference_givenstyle (scenedreamer.py:592-598)
    sky_avg = sky_attr.reshape(-1, 64) if sky_attr is not None else None
    win = _frame_window(voxel_id, depth2, raydirs) if (N == 1 and uniforms is None) else None
    if win is not None:
        bases, h0, w0, h, w = win
        # keyed on the tensor OBJECTS the tile loop hands over unchanged from tile to tile (a reshape would be a new object)
        keyt = list(bases) + [z, global_enc] + ([sky_attr] if sky_attr is not None else [])
        full, key = st.frame.lookup(keyt, st.epoch, (self.num_samples, float(self.sample_depth), float(self.dists_scale)))
        if full is None:
            st.stats['frame_launches'] += 1
            full = r.forward(bases[0].unsqueeze(0), bases[1].unsqueeze(0), bases[2].unsqueeze(0), cam_ori_t, z, global_enc,
                             sky_avg=sky_avg, want_samples=True, **kw)
            st.frame.store(key, keyt, full)
        else:
            st.stats['tile_hits'] += 1
        out = {k: full[k][:, h0:h0 + h, w0:w0 + w] for k in ('net_out', 'total_weight', 'weights', 'rand_depth', 'sky')}
        return _tuple12(out, sky_mask, sky_only_mask)
    out = r.forward(voxel_id.contiguous(), depth2.contiguous(), raydirs.contiguous(), cam_ori_t, z, global_enc,
                    uniforms=uniforms, sky_avg=sky_avg, want_samples=True, **kw)
    return _tuple12(out, sky_mask, sky_only_mask)


def fused_forward_global(self, net_out, z):
    """Replacement body of Base3DGenerator._forward_global (gancraft_base.py:588-603): RenderCNN + tanh on the tensor
    cores.  When `net_out` is a tile of the frame the fused per-pixel launch produced (the unmodified tile loop of
    inference_givenstyle), the CNN runs ONCE on the whole padded frame and every tile gets its window: the receptive
    radius is 4 px, the loop crops pad/2 = 15 px from every tile side (DESIGN.md section 1).  Calls that need gradients
    through the CNN (gen_update) keep the reference's cuDNN composition."""
    st = _state(self)
    reference = type(self)._sdb200_reference_forward_global
    needs_grad = torch.is_grad_enabled() and (net_out.requires_grad or (z is not None and z.requires_grad) or
                                              any(q.requires_grad for q in self.denoiser.parameters()))
    eng = None
    if enabled() and os.environ.get('SDB200_CNN', '1') != '0' and not needs_grad and z is not None and net_out.is_cuda and \
            net_out.dim() == 4 and net_out.shape[-1] == 64 and net_out.dtype == torch.float32:
        eng = st.get_cnn(self)
    if eng is None:
        st.stats['cnn_reference_calls'] += 1
        return reference(self, net_out, z)
    full = st.frame.out
    if full is not None and net_out.shape[0] == 1 and z.shape[0] == 1:
        base = full['net_out']
        if net_out._base is base and net_out.stride() == base.stride():
            HB, WB = base.shape[1], base.shape[2]
            off = net_out.storage_offset() - base.storage_offset()
            h0, rem = divmod(off, WB * 64)
            w0, rem = divmod(rem, 64)
            h, w = net_out.shape[1], net_out.shape[2]
            if rem == 0 and off >= 0 and h0 + h <= HB and w0 + w <= WB:
                if full.get('rgb_z') is not z:
                    st.stats['cnn_frame_launches'] += 1
                    full['rgb'], full['rgb_raw'] = eng.forward(base, z)
                    full['rgb_z'] = z
                else:
                    st.stats['cnn_tile_hits'] += 1
                return full['rgb'][:, :, h0:h0 + h, w0:w0 + w], full['rgb_raw'][:, :, h0:h0 + h, w0:w0 + w]
    st.stats['cnn_calls'] += 1
    return eng.forward(net_out, z)


SAMPLER_SPECULATION = 8          # most candidate poses judged per synchronisation (the depth adapts to the rejection rate)


def fused_get_batch(self, batch_size, device):
    """Replacement body of Generator._get_batch (scenedreamer.py:80-155): the training camera sampler.

    The reference draws a pose, raycasts it, and reads two statistics back to the host (mean first-hit depth, entropy of the
    first-hit labels: two blocking round trips per candidate) before deciding whether to keep it.  Here SAMPLER_SPECULATION
    candidates are drawn with the reference's OWN pose functions in the reference's order, raycast back to back, judged on
    the device by one small kernel each (ops.pose_stats) and read back with ONE synchronisation; the first accepted one wins
    and the host RNGs (torch, numpy) are rewound to their state right after that candidate was drawn.  The accepted poses,
    their order and the RNG streams afterwards are therefore exactly the reference's."""
    reference = type(self)._sdb200_reference_get_batch
    if not enabled() or os.environ.get('SDB200_SAMPLER', '1') == '0' or self.camera_sampler_type not in ('random', 'traditional') or \
            not torch.device(device).type == 'cuda':
        return reference(self, batch_size, device)
    import numpy as np
    from . import ops
    smod = sys.modules[type(self).__module__]
    camctl, mc_utils = smod.camctl, smod.mc_utils
    with torch.no_grad():
        if hasattr(self.voxel, 'sample_world'):
            self.voxel.sample_world(device)
        ids, deps, dirs, oris = [], [], [], []
        depth = max(1, min(SAMPLER_SPECULATION, int(getattr(self, '_sdb200_sampler_depth', 1))))
        for _ in range(batch_size):
            picked = None
            while picked is None:
                cands = []
                for _k in range(depth):
                    cam_res = self.cam_res                                           # scenedreamer.py:97-122, verbatim order of draws
                    cam_c = [(cam_res[0] - 1) / 2, (cam_res[1] - 1) / 2]
                    if self.camera_sampler_type == 'traditional' and torch.rand(1).item() > 0.5:
                        cam_ori_t, cam_dir_t, cam_up_t, cam_f = camctl.rand_camera_pose_tour(self.voxel)
                        cam_f = cam_f * (cam_res[1] - 1)
                    else:
                        cam_ori_t, cam_dir_t, cam_up_t = camctl.rand_camera_pose_thridperson2(self.voxel)
                        cam_f = 0.5 / np.tan(np.deg2rad(73 / 2) * (np.random.rand(1) * 0.5 + 0.5)) * (cam_res[1] - 1)
                    cam_res_crop = [self.crop_size[0] + self.pad, self.crop_size[1] + self.pad]
                    cam_c = mc_utils.rand_crop(cam_c, cam_res, cam_res_crop)
                    rng = (torch.get_rng_state(), np.random.get_state()) if _k + 1 < depth else None    # nothing drawn after the last
                    out = smod.voxlib.ray_voxel_intersection_perspective(self.voxel.voxel_t, cam_ori_t, cam_dir_t, cam_up_t, cam_f, cam_c,
                                                                         cam_res_crop, self.num_blocks_early_stop)
                    cands.append((out, cam_ori_t, rng, ops.pose_stats(out[0], out[1])))
                stats = torch.stack([c[3] for c in cands]).cpu()                     # the ONE synchronisation of this round
                for k, ((out, ori, rng, _s), (avg_depth, entropy)) in enumerate(zip(cands, stats.tolist())):
                    if self.camera_rej_avg_depth > 0 and avg_depth < self.camera_rej_avg_depth:
                        continue
                    if self.camera_min_entropy > 0 and entropy < self.camera_min_entropy:
                        continue
                    picked = (out, ori)
                    if rng is not None:
                        torch.set_rng_state(rng[0])                                  # forget the candidates drawn after the winner
                        np.random.set_state(rng[1])
                    break
                depth = max(1, depth // 2) if (picked is not None and k == 0) else min(SAMPLER_SPECULATION, depth * 2)
            ids.append(picked[0][0])
            deps.append(picked[0][1])
            dirs.append(picked[0][2])
            oris.append(picked[1])
        self._sdb200_sampler_depth = depth
        return torch.stack(ids, 0), torch.stack(deps, 0), torch.stack(dirs, 0), torch.stack(oris, 0).to(device), None


def _epoch_entry(name, fn):
    @functools.wraps(fn)
    def entry(self, *a, **k):
        _state(self).new_epoch()
        return fn(self, *a, **k)
    entry._sdb200_wrapped = fn
    return entry


# ------------------------------------------------------------------------------------------------
# installation
# ------------------------------------------------------------------------------------------------
def install(generator_cls, precision=DEFAULT_PRECISION):
    """Patch a reference `Generator` CLASS in place (idempotent)."""
    if not hasattr(generator_cls, '_forward_perpix'):
        raise TypeError('%r has no _forward_perpix: not a SceneDreamer generator' % (generator_cls,))
    if '_sdb200_reference_forward_perpix' in generator_cls.__dict__:
        return generator_cls
    generator_cls._sdb200_reference_forward_perpix = generator_cls._forward_perpix
    generator_cls._sdb200_precision = precision
    generator_cls._forward_perpix = fused_forward_perpix
    if os.environ.get('SDB200_ADAM', '1') != '0':
        optim.install_step_hook()                               # f2: the hash table's Adam step in one pass (optim.py)
    if '_get_batch' in generator_cls.__dict__ and hasattr(generator_cls, 'sample_camera'):
        generator_cls._sdb200_reference_get_batch = generator_cls._get_batch
        generator_cls._get_batch = fused_get_batch
    if hasattr(generator_cls, '_forward_global') and hasattr(generator_cls, '_forward_perpix_sub'):
        generator_cls._sdb200_reference_forward_global = generator_cls._forward_global
        generator_cls._forward_global = fused_forward_global
    for name in PUBLIC_ENTRIES:
        fn = generator_cls.__dict__.get(name)
        if fn is not None:
            setattr(generator_cls, name, _epoch_entry(name, fn))
    return generator_cls


def uninstall(generator_cls):
    ref = generator_cls.__dict__.get('_sdb200_reference_forward_perpix')
    if ref is None:
        return
    generator_cls._forward_perpix = ref
    del generator_cls._sdb200_reference_forward_perpix
    if '_sdb200_reference_get_batch' in generator_cls.__dict__:
        generator_cls._get_batch = generator_cls._sdb200_reference_get_batch
        del generator_cls._sdb200_reference_get_batch
    if '_sdb200_reference_forward_global' in generator_cls.__dict__:
        g = generator_cls._sdb200_reference_forward_global
        if '_forward_global' in generator_cls.__dict__:
            del generator_cls._forward_global                  # the method is inherited from Base3DGenerator
        del generator_cls._sdb200_reference_forward_global
    for name in PUBLIC_ENTRIES:
        fn = generator_cls.__dict__.get(name)
        if fn is not None and hasattr(fn, '_sdb200_wrapped'):
            setattr(generator_cls, name, fn._sdb200_wrapped)


def _unwrap(obj):
    """Generator instance inside WrappedModel / DDP (`.module`) / ModelAverage (`.averaged_model`) wrappers."""
    seen = 0
    while not hasattr(obj, '_forward_perpix') and seen < 8:
        nxt = getattr(obj, 'module', None)
        if nxt is None:
            nxt = getattr(obj, 'averaged_model', None)
        if nxt is None:
            break
        obj, seen = nxt, seen + 1
    if not hasattr(obj, '_forward_perpix'):
        raise TypeError('patch_generator: no SceneDreamer generator (object with _forward_perpix) inside %r' % type(obj))
    return obj


def patch_generator(gen, precision=DEFAULT_PRECISION):
    """Explicit route (one line after the generator is built): patches the CLASS of the wrapped generator."""
    g = _unwrap(gen)
    install(type(g), precision)
    return g


def invalidate(gen):
    """Forget packed weights / pre-blended table / frame results of this generator (call after editing weights
    through `.data`, which torch's version counter does not see, outside the public entry points)."""
    _state(_unwrap(gen)).new_epoch()


class _PatchingLoader(importlib.abc.Loader):
    def __init__(self, inner):
        self.inner = inner

    def create_module(self, spec):
        return self.inner.create_module(spec)

    def exec_module(self, module):
        self.inner.exec_module(module)
        ensure_installed()

    def __getattr__(self, name):
        return getattr(self.inner, name)


class _Finder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path, target=None):
        if fullname != TARGET_MODULE:
            return None
        for f in sys.meta_path:
            if f is self or not hasattr(f, 'find_spec'):
                continue
            spec = f.find_spec(fullname, path, target)
            if spec is not None and spec.loader is not None:
                spec.loader = _PatchingLoader(spec.loader)
                return spec
        return None


_finder = None
_installed = False


def ensure_installed():
    """Cheap check the drop-in ops make on every call: the reference imports `voxlib` from INSIDE the import of
    imaginaire.generators.scenedreamer (line 13), i.e. before `Generator` exists and after the module's loader has been
    picked -- too late for the import hook.  The first raycast / positional encoding of a run patches the class then;
    method lookup is dynamic, so even the `inference_givenstyle` call already in flight takes the fused path."""
    global _installed
    if _installed:
        return
    mod = sys.modules.get(TARGET_MODULE)
    if mod is not None and hasattr(mod, 'Generator'):
        if enabled():
            install(mod.Generator)
            pcg = sys.modules.get('imaginaire.model_utils.pcg_gen')
            if pcg is not None and hasattr(pcg, 'PCGVoxelGenerator') and os.environ.get('SDB200_WORLDGEN', '1') != '0':
                worldgen.install(pcg.PCGVoxelGenerator)             # f3: the scene's voxel world is built on the device
        _installed = True


def install_import_hook():
    """Called by dropin/voxlib.py when the reference imports `voxlib`: patch `Generator` as soon as
    imaginaire.generators.scenedreamer has been imported (or right now if it already is)."""
    global _finder
    ensure_installed()
    if _installed:
        return
    if _finder is None:
        _finder = _Finder()
        sys.meta_path.insert(0, _finder)
