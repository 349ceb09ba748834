"""Novel-view PSNR / SSIM of a checkpoint on a GlossySynthetic object's test views, on the GPU.

    python tools/eval_synthetic_nvs.py --cfg configs/shape/syn/bell.yaml [--ids 0 5 9]

Loads data/model/<name>/model.pth ({'step', 'network_state_dict', ...}) for a shape (stage I) or material (stage II) config
whose database_name is syn/<object>, and renders each test view at full resolution: by default the views of the first list of
configs/synthetic_split_128.pkl, read from data/GlossySynthetic/<object> (<id>-camera.pkl, <id>.png).  Stage I scores
render_image's `ray_rgb` against the ground-truth image at the checkpoint's step; stage II scores render_rays' `rgb_pr`
against its `rgb_gt`, the ground truth where the mesh is hit and zero elsewhere, as its validation does.  Scores are the exact
PSNR and the SSIM of nero_b200/metrics.py on the quantised images.  Writes the renders to data/nvs/<name>-<step>/<id>.png,
prints `<id> <psnr> <ssim>` per view and `<name>-<step> <mean psnr> <mean ssim>`, and appends that last line to
data/nvs.log.  Paths are relative to the working directory.  Real-data (real/) and custom (custom/) objects are refused:
their readers live in the training repository.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--cfg', type=str, required=True)
    parser.add_argument('--ids', type=str, nargs='+', default=None, help='view ids (default: the test split)')
    return parser.parse_args(argv)


def load_cfg(path):
    import yaml
    with open(path) as f:
        cfg = yaml.safe_load(f)
    if not isinstance(cfg, dict) or cfg.get('network') not in ('shape', 'material'):
        net = cfg.get('network') if isinstance(cfg, dict) else None
        raise SystemExit(f"eval_synthetic_nvs: {path} configures network '{net}'; novel views come from a shape or a material "
                         'network')
    db = str(cfg.get('database_name', ''))
    parts = db.split('/')
    if parts[0] != 'syn' or len(parts) != 2 or not parts[1]:
        raise SystemExit(f"eval_synthetic_nvs: database '{db}' is not a GlossySynthetic object (syn/<object>); real/ and custom/ "
                         'data are read by the training repository')
    return cfg


def render_view(network, kind, gt, pose, K, step):
    """(ground truth, render) of one view as uint8 CUDA [h, w, 3]: stage I (kind 'shape') render_image's gt_rgb / ray_rgb at
    `step`, stage II render_rays' rgb_gt / rgb_pr.  gt: uint8 [h, w, 3] numpy, pose [3, 4], K [3, 3]."""
    import numpy as np
    import torch
    from nero_b200 import metrics as M
    h, w = gt.shape[:2]
    info = {'imgs': torch.from_numpy(gt.astype(np.float32) / 255).permute(2, 0, 1)[None], 'Ks': torch.from_numpy(K)[None],
            'poses': torch.from_numpy(pose)[None]}
    if kind == 'material':
        out = network.render_rays(network._construct_ray_batch(info, 'cpu', False), h, w)
        rgb_gt, rgb_pr = out['rgb_gt'], out['rgb_pr']
    else:
        ray_batch, poses, _, h, w = network._construct_ray_batch(info)
        out = network.render_image(ray_batch, poses.float(), h, w, step)
        rgb_gt, rgb_pr = out['gt_rgb'], out['ray_rgb']
    return M.color_map_backward(rgb_gt.float()), M.color_map_backward(rgb_pr.float())


def main(argv=None):
    flags = parse(argv)
    cfg = load_cfg(flags.cfg)

    import numpy as np
    import torch
    from nero_b200 import evaluate as E
    from nero_b200 import metrics as M
    from nero_b200.relight import write_png

    root = os.path.join('data', 'GlossySynthetic', cfg['database_name'].split('/')[1])
    ids = flags.ids or E.split_test_ids()
    views = E.read_views(root, ids)
    if cfg['network'] == 'material':
        from nero_b200.material import NeROMaterialRenderer
        network = NeROMaterialRenderer(cfg, is_train=False)
    else:
        from nero_b200.renderer import NeROShapeRenderer
        network = NeROShapeRenderer(cfg, training=False)
    ckpt = torch.load(f'data/model/{cfg["name"]}/model.pth', map_location='cpu')
    step = ckpt['step']
    network.load_state_dict(ckpt['network_state_dict'])
    network = network.eval().cuda()
    print(f'successfully load {cfg["name"]} step {step}!')

    out_dir = os.path.join('data', 'nvs', f'{cfg["name"]}-{step}')
    os.makedirs(out_dir, exist_ok=True)
    scores = []
    for img_id, (pose, K, (h, w)) in zip(ids, views):
        gt = E.read_gt_image(root, img_id)
        if gt.shape[:2] != (h, w):
            raise SystemExit(f'eval_synthetic_nvs: {img_id}.png is {gt.shape[1]} x {gt.shape[0]}, expected {w} x {h}')
        q_gt, q_pr = render_view(network, cfg['network'], gt, pose, K, step)
        p, s = M.psnr(q_gt, q_pr), M.ssim(q_gt, q_pr)
        write_png(os.path.join(out_dir, f'{img_id}.png'), q_pr.cpu().numpy())
        scores.append((p, s))
        print(f'{img_id} {p:.4f} {s:.6f}')
    mp, ms = np.mean([p for p, _ in scores]), np.mean([s for _, s in scores])
    line = f'{cfg["name"]}-{step} {mp:.4f} {ms:.6f}'
    print(line)
    with open(os.path.join('data', 'nvs.log'), 'a') as f:
        f.write(line + '\n')
    return scores


if __name__ == '__main__':
    main()
