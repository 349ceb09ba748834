"""Drop-in replacements for the reference's renderers (network/renderer.py): same registry name, constructor,
cfg keys, forward(data) contract, output dictionaries and state_dict layout -- backed by the sm_90a kernels of
libnero_b200 instead of PyTorch ops.

    from nero_b200.renderer import name2renderer      # {'shape': NeROShapeRenderer, ...}
    net = name2renderer[cfg['network']](cfg).cuda()    # exactly what train/trainer.py:52 does
    outputs = net({'step': step})                      # train/trainer.py:128

Reference: network/renderer.py:63-647 (NeROShapeRenderer), :917-920 (name2renderer).
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .params import SDFParams, VarianceParams, NeRFParams, ShadingParams


class _RenderCoreFn(torch.autograd.Function):
    """render_core as ONE autograd node: forward and backward are kernel sequences (engine.py); parameter gradients
    are accumulated straight into the flat .grad buffer (they are not returned through autograd)."""

    @staticmethod
    def forward(ctx, engine, rays_o, rays_d, z_vals, human_poses, car, step, perm, *params):
        rgb, n_in, P = engine.render_core_forward(rays_o, rays_d, z_vals, human_poses, car, step, perm)
        w = engine.w
        gerr = w['GERR'][:n_in].clone() if n_in > 0 else torch.zeros(1, device=rgb.device)
        loss_occ = (w['OCC_LOSS'][0] / P).clone() if P > 0 else torch.zeros(1, device=rgb.device)
        n_reg = engine.n_reg
        sdf_vals = w['REG_SDF'][:n_reg, 0].clone() if n_reg > 0 else torch.zeros(0, device=rgb.device)
        ctx.engine, ctx.P, ctx.n_in, ctx.nparams, ctx.n_reg = engine, P, n_in, len(params), n_reg
        return rgb, gerr, loss_occ, sdf_vals

    @staticmethod
    def backward(ctx, d_rgb, d_gerr, d_occ, d_sdf_vals):
        e = ctx.engine
        if ctx.n_reg > 0:
            e.reg_backward(d_sdf_vals.contiguous())      # uses ABAR/dHa as scratch: must run before the main backward
        dscale = (d_occ.reshape(()) / ctx.P) if ctx.P > 0 else None
        e.render_core_backward(d_rgb, d_gerr if ctx.n_in > 0 else None, dscale)
        return (None,) * (8 + ctx.nparams)


class NeROShapeRenderer(nn.Module):
    default_cfg = {
        'std_net': 'default', 'std_act': 'exp', 'inv_s_init': 0.3, 'freeze_inv_s_step': None,
        'sdf_net': 'default', 'sdf_activation': 'none', 'sdf_bias': 0.5, 'sdf_n_layers': 8, 'sdf_freq': 6, 'sdf_d_out': 257,
        'geometry_init': True,
        'shader_config': {},
        'n_samples': 64, 'n_bg_samples': 32, 'inf_far': 1000.0, 'n_importance': 64, 'up_sample_steps': 4, 'perturb': 1.0,
        'anneal_end': 50000, 'train_ray_num': 512, 'test_ray_num': 1024, 'clip_sample_variance': True,
        'database_name': 'nerf_synthetic/lego/black_800',
        'test_downsample_ratio': True, 'downsample_ratio': 0.25, 'val_geometry': False,
        'rgb_loss': 'charbonier', 'apply_occ_loss': True, 'occ_loss_step': 20000, 'occ_loss_max_pn': 2048, 'occ_sdf_thresh': 0.01,
        'fixed_camera': False,
        # not a reference key: replay train_step as two captured CUDA graphs (nero_b200/graph.py) once step >= 1000
        'cuda_graph': False,
    }

    def __init__(self, cfg, training=True):
        super().__init__()
        self.cfg = {**self.default_cfg, **cfg}
        c = self.cfg
        if c['std_act'] != 'exp' or c['sdf_activation'] != 'none':
            raise NotImplementedError('only std_act=exp / sdf_activation=none (the values every shipped YAML uses)')
        self.sdf_network = SDFParams(d_out=c['sdf_d_out'], d_in=3, d_hidden=256, n_layers=c['sdf_n_layers'],
                                     skip_in=(c['sdf_n_layers'] // 2,), multires=c['sdf_freq'], bias=c['sdf_bias'],
                                     geometric_init=c['geometry_init'])
        self.deviation_network = VarianceParams(c['inv_s_init'])
        self.outer_nerf = NeRFParams()
        with torch.no_grad():
            self.outer_nerf.rgb_linear.bias.fill_(float(np.log(0.5)))
        self.color_network = ShadingParams(c['shader_config'])
        self._engine = None
        # extract_mesh.py:27 calls network.sdf_network.sdf(x): route it to the forward-only CUDA chain
        # (through a weak reference: a bound method stored on the child module would tie renderer <-> sdf_network into a
        # reference cycle that keeps the multi-GB workspaces alive until the cyclic GC runs, and would travel with deepcopy)
        import weakref
        me = weakref.ref(self)
        self.sdf_network.sdf = lambda x: me()._sdf_query(x)
        self._weights_dirty = True
        if training:
            self._init_dataset()

    def _sdf_query(self, x):
        with torch.no_grad():
            return self.engine.sdf_query(x)

    # ------------------------------------------------------------------ engine plumbing
    @property
    def engine(self):
        if self._engine is None:
            from .engine import ShapeEngine
            from . import ops as _ops
            _ops.require_cuda(self.deviation_network.variance.device, 'NeROShapeRenderer')
            self._engine = ShapeEngine(self, self.cfg)
        return self._engine

    def _apply(self, fn, *a, **k):
        self._engine = None      # parameters are re-created on .cuda()/.to(): rebuild the prepared layers lazily
        return super()._apply(fn, *a, **k)

    # ------------------------------------------------------------------ helpers kept from the reference contract
    def get_anneal_val(self, step):
        return 1.0 if self.cfg['anneal_end'] < 0 else float(np.min([1.0, step / self.cfg['anneal_end']]))

    @staticmethod
    def near_far_from_sphere(rays_o, rays_d):
        a = torch.sum(rays_d ** 2, dim=-1, keepdim=True)
        b = 2.0 * torch.sum(rays_o * rays_d, dim=-1, keepdim=True)
        mid = 0.5 * (-b) / a
        return torch.clamp(mid - 1.0, min=1e-3), mid + 1.0

    def get_human_coordinate_poses(self, poses):
        pn = poses.shape[0]
        cam_cen = (-poses[:, :, :3].permute(0, 2, 1) @ poses[:, :, 3:])[..., 0]
        if not self.cfg['fixed_camera']:
            cam_cen = torch.cat([cam_cen[:, :2], torch.zeros_like(cam_cen[:, :1])], -1)
        Y = torch.zeros([pn, 3], device=poses.device, dtype=poses.dtype)
        Y[:, 2] = -1.0
        Z = poses[:, 2, :3].clone()
        Z[:, 2] = 0
        Z = F.normalize(Z, dim=-1)
        X = torch.cross(Y, Z, dim=-1)
        R = torch.stack([X, Y, Z], 1)
        t = -R @ cam_cen[:, :, None]
        return torch.cat([R, t], -1)

    def compute_rgb_loss(self, rgb_pr, rgb_gt):
        kind = self.cfg['rgb_loss']
        if kind == 'l2':
            return torch.sum((rgb_pr - rgb_gt) ** 2, -1)
        if kind == 'l1':
            return torch.sum(F.l1_loss(rgb_pr, rgb_gt, reduction='none'), -1)
        if kind == 'smooth_l1':
            return torch.sum(F.smooth_l1_loss(rgb_pr, rgb_gt, reduction='none', beta=0.25), -1)
        if kind == 'charbonier':
            return torch.sqrt(torch.sum((rgb_gt - rgb_pr) ** 2, dim=-1) + 0.001)
        raise NotImplementedError

    # ------------------------------------------------------------------ the hot path
    def sample_ray(self, rays_o, rays_d, near, far, perturb, rand_inner=None, rand_bg=None):
        """z_vals [R, n_samples+n_importance+n_bg_samples] (network/renderer.py:403-443).  Random draws are made with
        torch in the reference's order (renderer.py:416, :422) unless passed in."""
        e = self.engine
        e.prepare_weights()
        self._weights_fresh = True      # consumed by the render_core call that follows in render()
        R = rays_o.shape[0]
        if perturb > 0 and rand_inner is None:
            rand_inner = torch.rand([R, 1], device=rays_o.device)
            rand_bg = torch.rand([R, self.cfg['n_bg_samples']], device=rays_o.device)
        if perturb <= 0:
            rand_inner = rand_bg = None
        with torch.no_grad():
            return e.sample_ray(rays_o.contiguous(), rays_d.contiguous(), near.contiguous(), far.contiguous(),
                                None if rand_inner is None else rand_inner.contiguous(),
                                None if rand_bg is None else rand_bg.contiguous())

    def render_core(self, rays_o, rays_d, z_vals, human_poses, cos_anneal_ratio=0.0, step=None, is_train=True, perm=None):
        e = self.engine
        if not getattr(self, '_weights_fresh', False):
            e.prepare_weights()          # render_core called on its own: fold weight-norm / rebuild operand images
        self._weights_fresh = False
        params = [p for p in self.parameters()]
        rgb, gerr, loss_occ, sdf_vals = _RenderCoreFn.apply(e, rays_o.contiguous(), rays_d.contiguous(), z_vals.contiguous(),
                                                  human_poses.contiguous(), float(cos_anneal_ratio), int(step), perm, *params)
        outputs = {'ray_rgb': rgb, 'gradient_error': gerr}
        inv_s = torch.exp(self.deviation_network.variance * 10.0).clip(1e-6, 1e6)
        if self.cfg['freeze_inv_s_step'] is not None and step < self.cfg['freeze_inv_s_step']:
            inv_s = inv_s.detach()
        outputs['std'] = torch.mean(1 / inv_s) if e.state['N_in'] > 0 else torch.zeros(1, device=rgb.device)
        if step < 1000:       # network/renderer.py:591-594 (consumed by InitSDFRegLoss, network/loss.py:98-120)
            outputs['sdf_pts'] = e.w['REG_PTS'][:e.n_reg, :3].clone()
            outputs['sdf_vals'] = sdf_vals
        if self.cfg['apply_occ_loss']:
            outputs['loss_occ'] = loss_occ
        if not is_train:      # network/renderer.py:602-604 -> compute_validation_info (:465-482)
            with torch.no_grad():
                outputs.update(e.validation_info(rays_o.contiguous(), rays_d.contiguous(), z_vals.contiguous(), human_poses.contiguous()))
        return outputs

    def render(self, rays_o, rays_d, near, far, human_poses, perturb_overwrite=-1, cos_anneal_ratio=0.0, is_train=True, step=None):
        perturb = self.cfg['perturb']
        if perturb_overwrite >= 0:
            perturb = perturb_overwrite
        z_vals = self.sample_ray(rays_o, rays_d, near, far, perturb)
        return self.render_core(rays_o, rays_d, z_vals, human_poses, cos_anneal_ratio=cos_anneal_ratio, step=step, is_train=is_train)

    # ------------------------------------------------------------------ dataset plumbing (host side, unchanged semantics)
    def _init_dataset(self):
        """network/renderer.py:136-165 -- needs the reference's `dataset` package on sys.path (drop-in scenario)."""
        from dataset.database import parse_database_name, get_database_split   # noqa: provided by the host repo
        from utils.base_utils import color_map_forward
        self.database = parse_database_name(self.cfg['database_name'])
        self.train_ids, self.test_ids = get_database_split(self.database)
        self.train_ids = np.asarray(self.train_ids)

        def info(ids):
            imgs = color_map_forward(np.stack([self.database.get_image(i) for i in ids], 0)).astype(np.float32)
            Ks = np.stack([self.database.get_K(i) for i in ids], 0).astype(np.float32)
            poses = np.stack([self.database.get_pose(i) for i in ids], 0).astype(np.float32)
            return {'imgs': torch.from_numpy(imgs).permute(0, 3, 1, 2), 'Ks': torch.from_numpy(Ks), 'poses': torch.from_numpy(poses)}
        self.train_imgs_info, self.test_imgs_info = info(self.train_ids), info(self.test_ids)
        self.train_num, self.test_num = len(self.train_ids), len(self.test_ids)
        self.train_batch, self.train_poses, self.tbn, _, _ = self._construct_ray_batch(self.train_imgs_info)
        self.train_poses = self.train_poses.float()
        self._shuffle_train_batch()

    def _shuffle_train_batch(self):
        """network/renderer.py:161-165.  The shuffled table lives in pinned host memory (train_step copies slices of it with
        non_blocking H2D); the two pinned buffers per key are allocated once and alternate, instead of re-pinning the
        whole table on every reshuffle."""
        self.train_batch_i = 0
        idx = torch.randperm(self.tbn, device='cpu')
        pin = torch.cuda.is_available()
        spare = getattr(self, '_train_batch_spare', None) or {}
        new = {}
        for k, v in self.train_batch.items():
            buf = spare.get(k)
            if buf is None or buf.shape != v.shape or buf.dtype != v.dtype:
                buf = torch.empty(v.shape, dtype=v.dtype, pin_memory=pin)
            torch.index_select(v, 0, idx, out=buf)
            new[k] = buf
        self._train_batch_spare = self.train_batch if all(not pin or v.is_pinned() for v in self.train_batch.values()) else {}
        self.train_batch = new

    def _construct_ray_batch(self, imgs_info, device='cpu'):
        imn, _, h, w = imgs_info['imgs'].shape
        ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing='ij')
        coords = torch.stack([xs, ys], -1).float()[None].repeat(imn, 1, 1, 1).reshape(imn, h * w, 2)
        coords = torch.cat([coords + 0.5, torch.ones(imn, h * w, 1)], 2)
        dirs = coords @ torch.inverse(imgs_info['Ks']).permute(0, 2, 1)
        imgs = imgs_info['imgs'].permute(0, 2, 3, 1).reshape(imn, h * w, 3)
        idxs = torch.arange(imn, dtype=torch.int64)[:, None, None].repeat(1, h * w, 1)
        rn = imn * h * w
        batch = {'dirs': dirs.float().reshape(rn, 3), 'rgbs': imgs.float().reshape(rn, 3), 'idxs': idxs.reshape(rn, 1)}
        return batch, imgs_info['poses'], rn, h, w

    def _process_ray_batch(self, ray_batch, poses):
        rays_d = ray_batch['dirs']
        idxs = ray_batch['idxs'][..., 0]
        rays_o = (poses[:, :, :3].permute(0, 2, 1) @ -poses[:, :, 3:])[idxs, :, 0]
        rays_d = (poses[idxs, :, :3].permute(0, 2, 1) @ rays_d.unsqueeze(-1))[..., 0]
        rays_d = F.normalize(rays_d, dim=-1)
        near, far = self.near_far_from_sphere(rays_o, rays_d)
        return rays_o, rays_d, near, far, self.get_human_coordinate_poses(poses)[idxs]

    def _poses_on_device(self, dev):
        p = getattr(self, '_train_poses_dev', None)
        if p is None or p[0] is not self.train_poses or p[1].device != dev:
            p = self._train_poses_dev = (self.train_poses, self.train_poses.to(dev))
        return p[1]

    def _train_step_graphed(self, step):
        """train_step with the render replayed from CUDA graphs: no host<->device synchronisation anywhere in the step."""
        from .graph import TrainStepGraphs
        rn = self.cfg['train_ray_num']
        dev = self.deviation_network.variance.device
        sl = slice(self.train_batch_i, self.train_batch_i + rn)
        dirs, idxs = self.train_batch['dirs'][sl], self.train_batch['idxs'][sl]
        rgbs = self.train_batch['rgbs'][sl].to(dev, non_blocking=True)
        key = TrainStepGraphs.key(self, rn, step)
        graphs = self.__dict__.setdefault('_graphs', {})
        g = graphs.get(key)
        if g is None:
            for k in [k for k in graphs if k[3] != key[3]]:      # workspaces were re-allocated: those graphs are stale
                del graphs[k]
            g = graphs[key] = TrainStepGraphs(self, rn, step)
        rgb, gmean, locc = g.run(dirs, idxs, self._poses_on_device(dev), self.get_anneal_val(step), list(self.parameters()))
        self.train_batch_i += rn
        if self.train_batch_i + rn >= self.tbn:
            self._shuffle_train_batch()
        outputs = {'ray_rgb': rgb, 'gradient_error': gmean}
        inv_s = torch.exp(self.deviation_network.variance * 10.0).clip(1e-6, 1e6)
        if self.cfg['freeze_inv_s_step'] is not None and step < self.cfg['freeze_inv_s_step']:
            inv_s = inv_s.detach()
        outputs['std'] = torch.mean(1 / inv_s)
        if self.cfg['apply_occ_loss']:
            outputs['loss_occ'] = locc
        outputs['loss_rgb'] = self.compute_rgb_loss(rgb, rgbs)
        return outputs

    def train_step(self, step):
        if self.cfg['cuda_graph'] and step >= 1000:
            return self._train_step_graphed(step)
        rn = self.cfg['train_ray_num']
        dev = self.deviation_network.variance.device
        batch = {k: v[self.train_batch_i:self.train_batch_i + rn].to(dev, non_blocking=True) for k, v in self.train_batch.items()}
        self.train_batch_i += rn
        if self.train_batch_i + rn >= self.tbn:
            self._shuffle_train_batch()
        rays_o, rays_d, near, far, hp = self._process_ray_batch(batch, self._poses_on_device(dev))
        outputs = self.render(rays_o, rays_d, near, far, hp, -1, self.get_anneal_val(step), is_train=True, step=step)
        outputs['loss_rgb'] = self.compute_rgb_loss(outputs['ray_rgb'], batch['rgbs'])
        return outputs

    def nvs(self, pose, K, h, w):
        """Novel-view colour image for a numpy pose [3,4] / intrinsics [3,3] (network/renderer.py:189-222): 1024-ray chunks,
        no jitter, step 300000.  Only `ray_rgb` is returned, so the validation extras of is_train=False are not computed."""
        dev = self.deviation_network.variance.device
        Kt = torch.from_numpy(np.asarray(K, np.float32)).unsqueeze(0).to(dev)
        poses = torch.from_numpy(np.asarray(pose, np.float32)).unsqueeze(0).to(dev)
        ys, xs = torch.meshgrid(torch.arange(h, device=dev), torch.arange(w, device=dev), indexing='ij')
        coords = torch.stack([xs, ys], -1).float().reshape(1, h * w, 2)
        coords = torch.cat([coords + 0.5, torch.ones(1, h * w, 1, device=dev)], 2)
        dirs = (coords @ torch.inverse(Kt).permute(0, 2, 1)).reshape(h * w, 3)
        idxs = torch.zeros(h * w, 1, dtype=torch.int64, device=dev)
        out = []
        with torch.no_grad():
            for ri in range(0, h * w, 1024):
                cur = {'dirs': dirs[ri:ri + 1024], 'idxs': idxs[ri:ri + 1024]}
                rays_o, rays_d, near, far, hp = self._process_ray_batch(cur, poses)
                out.append(self.render(rays_o, rays_d, near, far, hp, 0, 0, is_train=True, step=300000)['ray_rgb'].cpu().numpy())
        return np.reshape(np.concatenate(out, 0), [h, w, 3])

    def test_step(self, index, step):
        """Full-image validation render in chunks of `test_ray_num` rays (network/renderer.py:274-316).  Needs the host
        repo's `dataset` package (database access) exactly like the reference; the per-chunk render runs on the CUDA path."""
        import cv2
        from network.renderer import imgs_info_slice, imgs_info_downsample     # host repo helpers (pure tensor slicing)
        imgs_info = imgs_info_slice(self.test_imgs_info, torch.from_numpy(np.asarray([index], np.int64)))
        gt_depth, gt_mask = self.database.get_depth(self.test_ids[index])
        if self.cfg['test_downsample_ratio']:
            imgs_info = imgs_info_downsample(imgs_info, self.cfg['downsample_ratio'])
            h, w = gt_depth.shape
            dh, dw = int(self.cfg['downsample_ratio'] * h), int(self.cfg['downsample_ratio'] * w)
            gt_depth = cv2.resize(gt_depth, (dw, dh), interpolation=cv2.INTER_NEAREST)
            gt_mask = cv2.resize(gt_mask.astype(np.uint8), (dw, dh), interpolation=cv2.INTER_NEAREST)
        gt_depth, gt_mask = torch.from_numpy(gt_depth), torch.from_numpy(gt_mask.astype(np.int32))
        ray_batch, poses, rn, h, w = self._construct_ray_batch(imgs_info)
        return self.render_image(ray_batch, poses.float(), h, w, step, gt_depth, gt_mask)

    def render_image(self, ray_batch, poses, h, w, step, gt_depth=None, gt_mask=None):
        """The chunk loop of test_step (network/renderer.py:289-316) on an already constructed ray batch."""
        dev = self.deviation_network.variance.device
        poses = poses.to(dev)
        ray_batch = {k: v.to(dev) for k, v in ray_batch.items()}
        rn, trn = ray_batch['dirs'].shape[0], self.cfg['test_ray_num']
        keys = ['ray_rgb', 'gradient_error', 'normal', 'depth', 'diffuse_albedo', 'diffuse_light', 'diffuse_color', 'specular_albedo',
                'specular_light', 'specular_color', 'specular_ref', 'metallic', 'roughness', 'occ_prob', 'indirect_light', 'occ_prob_gt']
        if self.cfg['shader_config'].get('human_light', False) or self.engine.human:
            keys.append('human_light')
        outputs = {k: [] for k in keys}
        with torch.no_grad():
            for ri in range(0, rn, trn):
                cur = {k: v[ri:ri + trn] for k, v in ray_batch.items()}
                rays_o, rays_d, near, far, human_poses = self._process_ray_batch(cur, poses)
                o = self.render(rays_o, rays_d, near, far, human_poses, 0, 0, is_train=False, step=step)
                for k in keys:
                    outputs[k].append(o[k].detach())
        outputs = {k: torch.cat(v, 0) for k, v in outputs.items()}
        outputs['loss_rgb'] = self.compute_rgb_loss(outputs['ray_rgb'], ray_batch['rgbs'])
        outputs['gt_rgb'] = ray_batch['rgbs'].reshape(h, w, 3)
        outputs['ray_rgb'] = outputs['ray_rgb'].reshape(h, w, 3)
        if gt_depth is not None:
            outputs['gt_depth'], outputs['gt_mask'] = gt_depth.unsqueeze(-1), gt_mask.unsqueeze(-1)
        self.zero_grad()
        return outputs

    def forward(self, data):
        if 'eval' in data:        # network/renderer.py:608-627
            index = int(data['index']) if not isinstance(data['index'], int) else data['index']
            outputs = self.test_step(index, step=data['step'])
            if index == 0 and self.cfg['val_geometry']:       # network/renderer.py:618-623
                outputs['vertices'], outputs['triangles'] = self.extract_geometry(resolution=128, threshold=0.0)
            return outputs
        return self.train_step(data['step'])

    # ------------------------------------------------------------------ geometry / material export hooks
    def extract_fields(self, bound_min=(-1.0, -1.0, -1.0), bound_max=(1.0, 1.0, 1.0), resolution=128, outside_val=1.0):
        """The SDF sampled on a regular grid, 1.0 outside the unit sphere (extract_fields, network/field.py:1090-1104); the
        grid goes through the forward-only CUDA chain in x-slabs instead of 64^3 blocks."""
        return self._fill_grid(bound_min, bound_max, resolution, outside_val).cpu().numpy()

    GRID_SLAB_POINTS = 1 << 22

    def _fill_grid(self, bound_min, bound_max, resolution, outside_val=1.0):
        """The extract_fields grid as a device tensor [res,res,res], filled through engine.sdf_query in x-slabs of at most
        GRID_SLAB_POINTS points (a point's value does not depend on the slab it is queried in)."""
        dev = self.deviation_network.variance.device
        axes = [torch.linspace(float(bound_min[i]), float(bound_max[i]), resolution, device=dev) for i in range(3)]
        u = torch.empty(resolution, resolution, resolution, device=dev)
        step = max(1, self.GRID_SLAB_POINTS // (resolution * resolution))
        for x0 in range(0, resolution, step):
            xx, yy, zz = torch.meshgrid(axes[0][x0:x0 + step], axes[1], axes[2], indexing='ij')
            pts = torch.stack([xx, yy, zz], -1).reshape(-1, 3)
            with torch.no_grad():
                val = self.engine.sdf_query(pts)[:, 0]
            val = torch.where(torch.norm(pts, dim=-1) >= 1.0, torch.full_like(val, float(outside_val)), val)
            u[x0:x0 + step] = val.reshape(-1, resolution, resolution)
        return u

    def extract_mesh(self, resolution=512, threshold=0.0, bound_min=-1.0, bound_max=1.0):
        """extract_mesh.py / extract_geometry (network/field.py:1106-1113) on the GPU: the SDF grid stays on the device and goes
        through marching cubes (k_mcubes.cu, nero_b200.mesh).  Bounds are scalars or 3-vectors.  Returns numpy (vertices
        float64 [V,3] in world coordinates, triangles int64 [T,3]); triangles are wound towards the inside (SDF <= threshold)."""
        from .mesh import marching_cubes_cuda
        bmin = np.broadcast_to(np.asarray(bound_min, np.float32), (3,))
        bmax = np.broadcast_to(np.asarray(bound_max, np.float32), (3,))
        u = self._fill_grid(bmin, bmax, resolution)
        v, t = marching_cubes_cuda(u, threshold)
        del u
        vertices = v.cpu().numpy().astype(np.float64) / (resolution - 1.0) * (bmax - bmin)[None, :] + bmin[None, :]
        return vertices, t.cpu().numpy().astype(np.int64)

    def extract_geometry(self, bound_min=(-1.0, -1.0, -1.0), bound_max=(1.0, 1.0, 1.0), resolution=128, threshold=0.0):
        """extract_geometry (network/field.py:1106-1113): marching cubes on the field; the cubes stay third party (PyMCubes,
        as in the reference) and are imported here, where they are needed."""
        u = self.extract_fields(bound_min, bound_max, resolution)
        import mcubes                 # noqa: the host repo's dependency (requirements.txt of the reference)
        vertices, triangles = mcubes.marching_cubes(u, threshold)
        bmin, bmax = np.asarray(bound_min, np.float32), np.asarray(bound_max, np.float32)
        vertices = vertices / (resolution - 1.0) * (bmax - bmin)[None, :] + bmin[None, :]
        return vertices, triangles

    def predict_materials(self, xyz=None, batch_size=8192):
        """Per-vertex metallic / roughness / albedo of the extracted mesh (network/renderer.py:629-647): SDF feature vector ->
        color_network.predict_materials (field.py:653-657).  `xyz` [V,3] supplies the vertices directly; by default they are
        read from data/meshes/{cfg['name']}-300000.ply like the reference does."""
        if xyz is None:
            from .material import read_ply
            xyz, _ = read_ply(f"data/meshes/{self.cfg['name']}-300000.ply")
        dev = self.deviation_network.variance.device
        xyz = torch.as_tensor(np.asarray(xyz, np.float32) if not torch.is_tensor(xyz) else xyz).to(dev)
        e = self.engine
        e.prepare_weights()
        outs = {'metallic': [], 'roughness': [], 'albedo': []}
        with torch.no_grad():
            for vi in range(0, xyz.shape[0], batch_size):
                m, r, a = e.materials_query(xyz[vi:vi + batch_size])
                outs['metallic'].append(m.cpu().numpy())
                outs['roughness'].append(r.cpu().numpy())
                outs['albedo'].append(a.cpu().numpy())
        return {k: np.concatenate(v, 0) for k, v in outs.items()}

    def export_lighting(self, width=1024, height=512, ssaa=4, center=(0.0, 0.0, 0.0), trans=False, kappa_inv=(0.0, 0.1, 0.25, 0.5, 1.0),
                        max_rows=None):
        """Stage I's pre-filtered outer light as CUDA float32 [height, width, 3] maps in relight's convention, one per kappa_inv
        (nero_b200/envmap.py): outer_light(IDE(d, k)) (field.py:554-589); k = 1 is the diffuse light, smaller k the specular
        light at roughness k.  -> {k: map}.  With sphere_direction the light is seen from `center`; trans=True gives the maps
        tools/relight.py --trans expects."""
        from . import envmap as EM
        c = self.color_network.cfg
        ol = EM.OuterLight(self.color_network.outer_light, c['light_exp_max'], 'stage1' if c['sphere_direction'] else None)
        frame = EM.trans_frame(trans)
        return {float(k): ol.map(width, height, ssaa, float(k), center, frame, max_rows or EM.MAX_ROWS) for k in kappa_inv}


def _material_renderer(*a, **k):
    from .material import NeROMaterialRenderer
    return NeROMaterialRenderer(*a, **k)


name2renderer = {'shape': NeROShapeRenderer, 'material': _material_renderer}   # network/renderer.py:917-920
