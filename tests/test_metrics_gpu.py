"""Image metrics on the GPU: quantisation, the exact PSNR and the SSIM map against the numpy / scipy oracle bit for bit,
determinism and batch independence, the refusals, the validation drop-ins on real render outputs, and
tools/eval_synthetic_nvs.py end to end for both stages."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import make_golden_metrics as G
import nero_oracle as O
import nero_oracle_mat as OMat
import nero_oracle_metrics as OM
from nero_b200 import metrics as M
from nero_b200 import ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'metrics_reference.npz')
cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()


def noisy_pair(seed, shape, noise=25):
    rng = np.random.RandomState(seed)
    gt = rng.randint(0, 256, shape).astype(np.uint8)
    pr = np.clip(gt.astype(np.int64) + rng.randint(-noise, noise + 1, shape), 0, 255).astype(np.uint8)
    return gt, pr


def test_quantisation_is_numpy_color_map_backward():
    g = np.load(GOLD)
    assert np.array_equal(M.color_map_backward(cu(g['quant_in'])).cpu().numpy(), g['quant_out'])
    rng = np.random.RandomState(1)
    x = np.concatenate([rng.uniform(-2, 3, 1 << 20), np.arange(-300, 600) / 255.0, (np.arange(256) + 0.5) / 255.0]).astype(np.float32)
    x = np.concatenate([x, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf))])
    x[::997] = np.nan
    x[1::991] = np.inf
    x[2::983] = -np.inf
    q = M.color_map_backward(cu(x).reshape(-1, 3)).cpu().numpy().reshape(-1)
    assert np.array_equal(q, OM.color_map_backward(x))
    with np.errstate(invalid='ignore'):
        assert np.array_equal(q, np.clip(x * 255, 0, 255).astype(np.uint8))


def test_psnr_is_exact():
    g = np.load(GOLD)
    for p in g['pairs']:
        gt, pr = G.image_pair(*p)
        v = M.psnr(cu(gt), cu(pr))
        assert isinstance(v, float) and v == OM.psnr_exact(gt, pr)
        B = np.stack([gt, pr, gt, 255 - gt])
        sse = torch.empty(4, 3, dtype=torch.int64, device='cuda')
        ops.K('nero_metrics_sse', cu(B), cu(np.stack([pr, pr, gt, gt])), 4, *gt.shape, sse)
        want = [OM.sse(gt, pr), OM.sse(pr, pr), OM.sse(gt, gt), OM.sse(255 - gt, gt)]
        assert np.array_equal(sse.cpu().numpy(), np.stack(want))
        assert M.psnr(cu(gt), cu(gt)) == np.inf
    gt, pr = noisy_pair(3, (37, 53, 1))
    assert M.psnr(cu(gt), cu(pr)) == OM.psnr_exact(gt, pr)
    batch = M.psnr(cu(np.stack([gt, gt])), cu(np.stack([pr, gt])))
    assert batch.dtype == np.float64 and batch[0] == OM.psnr_exact(gt, pr) and batch[1] == np.inf


@pytest.mark.parametrize('h,w', [(11, 11), (11, 12), (37, 53), (800, 800)])
@pytest.mark.parametrize('c', [1, 3])
def test_ssim_map_is_bit_identical_to_the_oracle(h, w, c):
    gt, pr = noisy_pair(h * 7 + w + c, (h, w, c))
    score, smap = M.ssim(cu(gt), cu(pr), full=True)
    osmap, ochan = OM.ssim_map(gt, pr)
    assert smap.dtype == torch.float64 and tuple(smap.shape) == (h, w, c)
    assert np.array_equal(smap.cpu().numpy(), osmap)
    assert abs(score - OM.ssim(gt, pr)) <= 1e-12
    assert score == M.ssim(cu(gt), cu(pr))
    one, ones = M.ssim(cu(gt), cu(gt), full=True)
    assert one == 1.0 and (ones == 1.0).all()


def test_ssim_is_deterministic_and_batch_independent():
    pairs = [noisy_pair(s, (64, 48, 3), 10 * s) for s in range(1, 5)]
    gts, prs = cu(np.stack([p[0] for p in pairs])), cu(np.stack([p[1] for p in pairs]))
    s1, m1 = M.ssim(gts, prs, full=True)
    s2, m2 = M.ssim(gts, prs, full=True)
    assert np.array_equal(s1, s2) and torch.equal(m1, m2)
    for i, (gt, pr) in enumerate(pairs):
        alone, malone = M.ssim(cu(gt), cu(pr), full=True)
        assert alone == s1[i] and torch.equal(malone, m1[i])
        assert abs(alone - OM.ssim(gt, pr)) <= 1e-12
    # more images than one workspace holds: the groups give the same bits
    old = M.MAX_WORK
    try:
        M.MAX_WORK = 2 * (5 * 64 * 48 * 3 + 3 * 64)
        s3, m3 = M.ssim(gts, prs, full=True)
    finally:
        M.MAX_WORK = old
    assert np.array_equal(s1, s3) and torch.equal(m1, m3)


def test_refusals():
    a = cu(np.zeros((16, 16, 3), np.uint8))
    for f in (M.psnr, M.ssim):
        with pytest.raises(RuntimeError):
            f(a.cpu(), a.cpu())
        with pytest.raises(ValueError):
            f(a, a[:, :15])
        with pytest.raises(ValueError):
            f(a.float(), a.float())
        with pytest.raises(ValueError):
            f(a[None, ..., None], a[None, ..., None])
        with pytest.raises(ValueError):
            f(a[..., :1].repeat(1, 1, 5), a[..., :1].repeat(1, 1, 5))
    with pytest.raises(ValueError):
        M.ssim(a[:10], a[:10])
    with pytest.raises(ValueError):
        M.ssim(a[:, :10], a[:, :10])
    with pytest.raises(ValueError):
        M.color_map_backward(torch.zeros(4, dtype=torch.float64, device='cuda'))
    with pytest.raises(RuntimeError):
        M.color_map_backward(torch.zeros(4))
    work = torch.empty(5 * 16 * 16 * 3 + 3 * 16, dtype=torch.float64, device='cuda')
    out = torch.empty(3, dtype=torch.float64, device='cuda')
    for win in (10, 17, 1):
        with pytest.raises(RuntimeError):
            ops.K('nero_metrics_ssim', a, a, 1, 16, 16, 3, win, M.COV_NORM, M.C1, M.C2, work, None, out)
    with pytest.raises(RuntimeError):
        ops.K('nero_metrics_sse', a, a, 1, 16, 16, 5, out)


# ------------------------------------------------------------------------------------------------ the drop-ins
def look_at(c, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    c = np.asarray(c, np.float64)
    z = np.asarray(target, np.float64) - c
    z /= np.linalg.norm(z)
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 0)
    return np.concatenate([R, (-R @ c)[:, None]], 1).astype(np.float32)


H, W = 24, 32
K = np.asarray([[40.0, 0, 16.0], [0, 40.0, 12.0], [0, 0, 1]], np.float32)
CAMS = [(2.2, 0.4, 0.6), (-0.7, 1.9, -0.9), (0.3, -1.2, 2.1)]
SHAPE_CFG = {'n_samples': 32, 'n_importance': 32}
SHADER_CFG = {'human_lights': False, 'diffuse_sample_num': 16, 'specular_sample_num': 16}


def stage1_net():
    from nero_b200 import params as P
    from nero_b200.renderer import NeROShapeRenderer
    sd = O.perturb_params(P.build_shape_state_dict(SHAPE_CFG, seed=6033), seed=11)
    net = NeROShapeRenderer(SHAPE_CFG, training=False)
    net.load_state_dict(sd)
    return net.cuda(), sd


def stage2_net(mesh):
    from nero_b200 import params as P
    from nero_b200.material import NeROMaterialRenderer
    sd = O.perturb_params(P.build_material_state_dict(SHADER_CFG, seed=6033), seed=11)
    net = NeROMaterialRenderer({'shader_cfg': SHADER_CFG, 'database_name': 'syn/ball'}, is_train=False, mesh=mesh)
    net.load_state_dict(sd)
    return net.cuda(), sd


def camera_info(i, gt):
    return {'imgs': torch.from_numpy(gt.astype(np.float32) / 255).permute(2, 0, 1)[None], 'Ks': torch.from_numpy(K)[None],
            'poses': torch.from_numpy(look_at(CAMS[i]))[None]}


def capture_montage(monkeypatch):
    seen = []
    write = M.write_montage

    def record(path, img):
        seen.append((path, img.cpu().numpy()))
        write(path, img)
    monkeypatch.setattr(M, 'write_montage', record)
    return seen


def check_outputs(out, gt, pr, montage, seen, path):
    import cv2
    assert set(out) == {'psnr', 'ssim'} and out['psnr'].shape == out['ssim'].shape == (1,)
    assert out['psnr'].dtype == out['ssim'].dtype == np.float64
    assert out['psnr'][0] == OM.psnr_exact(gt, pr) and abs(out['ssim'][0] - OM.ssim(gt, pr)) <= 1e-12
    assert len(seen) == 1 and seen[0][0] == path and np.array_equal(seen[0][1], montage)
    img = cv2.imread(path)
    assert img is not None and img.shape == montage.shape


def test_shape_render_metrics(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    seen = capture_montage(monkeypatch)
    net, _ = stage1_net()
    gt = np.random.RandomState(2).randint(0, 256, (H, W, 3)).astype(np.uint8)
    ray_batch, poses, _, h, w = net._construct_ray_batch(camera_info(0, gt))
    data_pr = net.render_image(ray_batch, poses.float(), h, w, 30000)
    out = M.name2metrics['shape_render']({})(data_pr, None, 30000, data_index=3, model_name='bell')
    host = {k: v.detach().cpu().numpy() for k, v in data_pr.items()}
    assert np.array_equal(OM.color_map_backward(host['gt_rgb']), gt)
    check_outputs(out, gt, OM.color_map_backward(host['ray_rgb']), OM.shape_montage(host), seen,
                  os.path.join('data', 'train_vis', 'bell', '30000-index-3.jpg'))
    assert M.name2key_metrics['psnr']({'psnr': np.asarray([out['psnr'][0], 20.0])}) == np.mean([out['psnr'][0], 20.0])


def test_material_render_metrics(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    seen = capture_montage(monkeypatch)
    net, _ = stage2_net(OMat.test_scene(2))
    gt = np.random.RandomState(4).randint(0, 256, (H, W, 3)).astype(np.uint8)
    data_pr = net.render_rays(net._construct_ray_batch(camera_info(1, gt), 'cpu', False), H, W)
    out = M.name2metrics['mat_render']({})(data_pr, None, 7, data_index=0, model_name='bell_mat')
    host = {k: v.detach().cpu().numpy() for k, v in data_pr.items()}
    hit = host['rgb_gt'].any(-1)
    assert 0 < hit.sum() < H * W
    check_outputs(out, OM.color_map_backward(host['rgb_gt']), OM.color_map_backward(host['rgb_pr']), OM.material_montage(host),
                  seen, os.path.join('data', 'train_vis', 'bell_mat', '7-index-0.jpg'))


# ------------------------------------------------------------------------------------------------ the tool
def make_object(ws, gts):
    """data/GlossySynthetic/ball with views 0..2 (camera pickles, RGBA PNGs of the given RGB images) and a split listing them
    in the order 2, 0, 1."""
    import cv2
    root = ws / 'data' / 'GlossySynthetic' / 'ball'
    os.makedirs(root, exist_ok=True)
    for i, gt in enumerate(gts):
        with open(root / f'{i}-camera.pkl', 'wb') as f:
            pickle.dump([look_at(CAMS[i]).astype(np.float64), K.astype(np.float64)], f)
        alpha = np.full((H, W, 1), 255 - i, np.uint8)
        cv2.imwrite(str(root / f'{i}.png'), np.concatenate([gt[..., ::-1], alpha], -1))
    os.makedirs(ws / 'configs', exist_ok=True)
    with open(ws / 'configs' / 'synthetic_split_128.pkl', 'wb') as f:
        pickle.dump([np.asarray(['2', '0', '1']), []], f)


@pytest.mark.parametrize('stage', ['shape', 'material'])
def test_tool_end_to_end(tmp_path, stage):
    import cv2
    import yaml
    from nero_b200.mesh import write_ply
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import eval_synthetic_nvs as T
    step = 123
    if stage == 'shape':
        net, sd = stage1_net()
        cfg = dict(SHAPE_CFG, name='nvs1', network='shape', database_name='syn/ball')
    else:
        mesh = OMat.test_scene(2)
        net, sd = stage2_net(mesh)
        write_ply(str(tmp_path / 'mesh.ply'), *mesh)
        cfg = {'name': 'nvs2', 'network': 'material', 'database_name': 'syn/ball', 'mesh': str(tmp_path / 'mesh.ply'),
               'shader_cfg': SHADER_CFG}
    os.makedirs(tmp_path / 'data' / 'model' / cfg['name'])
    torch.save({'step': step, 'network_state_dict': sd}, tmp_path / 'data' / 'model' / cfg['name'] / 'model.pth')
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    # view 0: the model's own quantised render (stage II: black where the mesh is missed) -> inf / 1.0;
    # views 1 and 2: that render with noise, and noise alone
    rng = np.random.RandomState(8)
    blank = np.zeros((H, W, 3), np.uint8)
    own = [T.render_view(net, stage, blank, look_at(CAMS[i]), K, step)[1].cpu().numpy() for i in range(3)]
    gts = [own[0], np.clip(own[1].astype(int) + rng.randint(-20, 21, own[1].shape), 0, 255).astype(np.uint8),
           rng.randint(0, 256, (H, W, 3)).astype(np.uint8)]
    make_object(tmp_path, gts)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    run = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'eval_synthetic_nvs.py'), '--cfg', 'cfg.yaml'], cwd=tmp_path,
                         env=env, capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    lines = run.stdout.strip().split('\n')[-4:]
    got = {l.split()[0]: l.split()[1:] for l in lines[:3]}
    assert list(got) == ['2', '0', '1']
    assert got['0'] == ['inf', '1.000000']
    ps, ss = [], []
    for i in ('2', '0', '1'):
        pr = cv2.imread(str(tmp_path / 'data' / 'nvs' / f'{cfg["name"]}-{step}' / f'{i}.png'), cv2.IMREAD_UNCHANGED)[..., ::-1]
        assert np.array_equal(pr, own[int(i)])
        gt = gts[int(i)]
        if stage == 'material':      # render_rays' ground truth is zero where the mesh is missed
            gt = T.render_view(net, stage, gt, look_at(CAMS[int(i)]), K, step)[0].cpu().numpy()
        ps.append(OM.psnr_exact(gt, pr))
        ss.append(OM.ssim(gt, pr))
        assert got[i] == [f'{ps[-1]:.4f}', f'{ss[-1]:.6f}'], (i, got[i], ps[-1], ss[-1])
    line = f'{cfg["name"]}-{step} {np.mean(ps):.4f} {np.mean(ss):.6f}'
    assert lines[3] == line
    assert (tmp_path / 'data' / 'nvs.log').read_text() == line + '\n'
    sub = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'eval_synthetic_nvs.py'), '--cfg', 'cfg.yaml', '--ids', '1'],
                         cwd=tmp_path, env=env, capture_output=True, text=True)
    assert sub.returncode == 0, sub.stderr
    assert sub.stdout.strip().split('\n')[-2].split()[1:] == got['1']
