"""CPU: the normal-map byte encoding, the oracle bake of a coarse icosphere against a fine one, the PNG round trip, the
texel table with and without a map, the oracle's normal-mapped shading with a map that falls back everywhere, and the
argument errors of tools/relight.py --normal-map and tools/bake_normal_map.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

import nero_oracle_normalmap as ON
import nero_oracle_relight as OR
import nero_oracle_relight_tex as ORT
from nero_b200 import normalmap as NM
from nero_b200 import relight as RL
from nero_b200 import synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, 'tools')


def mc_wound_icosphere(subdiv):
    """synthetic.icosphere wound like marching-cubes meshes: cross(e1, e2) pointing into the solid."""
    v, f = synthetic.icosphere(subdiv, 0.5)
    return v, np.ascontiguousarray(f[:, [0, 2, 1]])


def test_encoding_round_trips_every_byte():
    k = np.arange(256, dtype=np.uint8)
    assert np.array_equal(NM.encode(NM.decode(k)), k)
    assert np.array_equal(ON.encode(ON.decode(k)), k)
    assert np.array_equal(NM.decode(k), ON.decode(k))
    assert NM.decode(0) == -1 and NM.decode(255) == 1
    n = np.random.RandomState(1).randn(4096, 3).astype(np.float32) * 0.7
    assert np.array_equal(NM.encode(n), ON.encode(n))
    assert np.array_equal(NM.encode([[-2.0, 0.0, 2.0]]), [[0, 128, 255]])     # clamped; 0 encodes to 128


def test_oracle_vertex_normals_are_outward_and_order_fixed():
    v, f = mc_wound_icosphere(2)
    n = ON.vertex_normals(v, f)
    r = v / np.linalg.norm(v, axis=1, keepdims=True)
    assert np.degrees(np.arccos(np.clip((n * r).sum(1), -1, 1))).max() < 2.0     # 1.35 degrees at subdivision 2
    # an unreferenced vertex gives (0, 0, 0) and changes no other normal
    v2 = np.concatenate([v, [[9, 9, 9]]]).astype(np.float32)
    n2 = ON.vertex_normals(v2, f)
    assert (n2[-1] == 0).all() and np.array_equal(n2[:-1], n)


# Max angle between the baked normal and the radial direction at the hit point, measured with the oracle below: 0.33
# degrees (the fine sphere's own vertex normals are within 0.34 degrees of radial).
MAX_RADIAL_DEG = 0.5


def test_oracle_bake_of_a_coarse_sphere_recovers_the_fine_sphere():
    """The 80-triangle icosphere baked against the 5120-triangle one: the coarse faces lie up to 0.025 inside the fine
    surface, so the cage distance is 0.05; every ray hits, and the normals are the fine sphere's (radial) ones."""
    from nero_b200.texmap import uv_atlas
    lv, lf = mc_wound_icosphere(1)
    dv, df = mc_wound_icosphere(4)
    vt, ft = uv_atlas(lv, lf, 48, 48, 2)
    b = ON.bake_texels(lv, lf, vt, ft, dv, df, 48, 48, distance=0.05)
    assert b['texel'].size > 500
    assert b['hit'].all() and not b['tie'].any()
    p = b['point'] + np.float32(0.05) * b['cage'] - b['t'][:, None] * b['cage']
    r = p / np.linalg.norm(p, axis=1, keepdims=True)
    ang = np.degrees(np.arccos(np.clip((b['normal'] * r).sum(1), -1, 1)))
    print(f'coarse -> fine sphere: {b["texel"].size} texels, max angle to radial {ang.max():.3f} degrees')
    assert ang.max() < MAX_RADIAL_DEG
    # the coarse mesh's own interpolated normals are up to ~16 degrees off radial: the bake is what brings them back
    pc = b['point'] / np.linalg.norm(b['point'], axis=1, keepdims=True)
    flat = ON.face_areas32(lv, lf)[b['owner'].reshape(-1)[b['texel']]]
    flat = flat / np.linalg.norm(flat, axis=1, keepdims=True)
    assert np.degrees(np.arccos(np.clip((flat * pc).sum(1), -1, 1))).max() > 5
    img, stats, _ = ON.bake(lv, lf, vt, ft, dv, df, 24, 2, 0.05)
    assert img.shape == (24, 24, 3) and stats == {'covered': b['texel'].size, 'hits': b['texel'].size, 'misses': 0}


def test_png_round_trip(tmp_path):
    rng = np.random.RandomState(3)
    img = rng.randint(0, 256, (17, 29, 3)).astype(np.uint8)
    path = str(tmp_path / 'normal_0.png')
    NM.write_normal_map(path, img)
    back = NM.read_normal_map(path)
    assert back.shape == (17, 29, 3) and back.dtype == np.float32
    assert np.array_equal(NM.encode(back), img)
    assert np.array_equal(back, NM.decode(img))            # linear: no sRGB transfer, no renormalisation
    with pytest.raises(ValueError, match='missing'):
        NM.read_normal_map(str(tmp_path / 'nope.png'))


def old_texel_table(albedo, metallic, roughness):
    H, W = albedo.shape[:2]
    t = np.zeros((H, W, 8), np.float32)
    t[..., :3], t[..., 3], t[..., 4] = albedo, metallic.reshape(H, W), roughness.reshape(H, W)
    return t


def test_texel_table_layout():
    rng = np.random.RandomState(5)
    vt, ft = rng.rand(6, 2).astype(np.float32), np.asarray([[0, 1, 2], [3, 4, 5]], np.int32)
    alb, met, rough = rng.rand(5, 7, 3), rng.rand(5, 7), rng.rand(5, 7, 1)
    plain = RL.UVMaterials(vt, ft, alb, met, rough).texel_table()
    assert plain.tobytes() == old_texel_table(alb.astype(np.float32), met.astype(np.float32), rough.astype(np.float32)).tobytes()
    nrm = rng.randn(5, 7, 3).astype(np.float32)
    mapped = RL.UVMaterials(vt, ft, alb, met, rough, normal=nrm).texel_table()
    assert np.array_equal(mapped[..., :5], plain[..., :5]) and np.array_equal(mapped[..., 5:], nrm)
    with pytest.raises(ValueError, match='normal map has shape'):
        RL.UVMaterials(vt, ft, alb, met, rough, normal=nrm[:4])
    with pytest.raises(ValueError, match='non-finite'):
        RL.UVMaterials(vt, ft, alb, met, rough, normal=np.full((5, 7, 3), np.nan, np.float32))


def test_oracle_nmap_render_with_a_zero_map_is_the_textured_render():
    """A map of zeros falls back to the flat normal everywhere, and then the normal-mapped rule is the textured one."""
    import nero_oracle_mat as OM
    verts, tris = OM.test_scene(1)
    rng = np.random.RandomState(2)
    vt = rng.rand(verts.shape[0], 2)
    tex = np.zeros((6, 8, 8))
    tex[..., :3], tex[..., 3], tex[..., 4] = rng.rand(6, 8, 3), rng.rand(6, 8), 0.3 + 0.7 * rng.rand(6, 8)
    tables = RL.env_tables(np.exp(rng.randn(8, 16, 3)).astype(np.float32))
    pose, K = RL.relight_poses(3, 20.0, 30.0, 2.0)[1], RL.blender_default_K(10, 10)
    a = ORT.render(verts, tris, (vt, tris, tex), tables, pose, K, 10, 10, 1, 3, seed=4)
    b = ON.render(verts, tris, (vt, tris, tex), tables, pose, K, 10, 10, 1, 3, seed=4)
    assert a[..., 3].any() and np.array_equal(a, b)
    # a map of random directions changes the colours but not the coverage
    tex2 = tex.copy()
    tex2[..., 5:] = OR.normalize(rng.randn(6, 8, 3))
    c = ON.render(verts, tris, (vt, tris, tex2), tables, pose, K, 10, 10, 1, 3, seed=4)
    assert np.array_equal(c[..., 3], a[..., 3]) and not np.array_equal(c[..., :3], a[..., :3])


def run_tool(name, args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, os.path.join(TOOLS, name)] + args, cwd=cwd, env=env, capture_output=True, text=True)


def test_relight_tool_argument_errors(tmp_path):
    from nero_b200.texmap import write_textured_obj
    r = run_tool('relight.py', ['--mesh', 'm.ply', '--material', 'mat', '--hdr', 'e.hdr', '--name', 'x', '--normal-map', 'n.png'], tmp_path)
    assert r.returncode == 2 and '--normal-map needs --obj' in r.stderr, r.stderr
    verts, tris = mc_wound_icosphere(0)
    rng = np.random.RandomState(0)
    vt, ft = rng.rand(3 * tris.shape[0], 2).astype(np.float32), np.arange(3 * tris.shape[0], dtype=np.int32).reshape(-1, 3)
    grey = np.full((8, 8, 3), 128, np.uint8)
    write_textured_obj(str(tmp_path / 'n2m'), verts, tris, vt, ft, (grey, grey, grey))
    NM.write_normal_map(str(tmp_path / 'n2m' / 'normal_0.png'), np.full((4, 4, 3), 128, np.uint8))
    r = run_tool('relight.py', ['--obj', 'n2m/mesh_0.obj', '--normal-map', 'n2m/normal_0.png', '--hdr', 'e.hdr', '--name', 'x'], tmp_path)
    assert r.returncode != 0 and 'n2m/normal_0.png' in r.stderr and '4x4' in r.stderr and '8x8' in r.stderr, r.stderr
    assert not (tmp_path / 'data' / 'relight' / 'x' / '0.png').exists()
    r = run_tool('bake_normal_map.py', ['--obj', 'n2m/mesh_0.obj', '--detail', 'd.ply', '--size', '0'], tmp_path)
    assert r.returncode == 2 and '--size 0' in r.stderr, r.stderr
