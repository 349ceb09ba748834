"""Generate tests/golden/texmap_*.npz by running the UNMODIFIED reference texture_mapper of extract_materials_texture_map.py on
CPU.

    python oracle/make_golden_texmap.py [<path to the reference checkout>]

What runs unmodified (through ref_shim, .cuda() mapped to the CPU): texture_mapper / _export_obj, NeROMaterialRenderer's
constructor, MCShadingNetwork.predict_materials_n2m (fp32 on the CPU: autocast does not apply), linear_to_srgb, scipy's
binary_dilation / binary_erosion, sklearn's kd-tree NearestNeighbors, cv2.cvtColor / cv2.resize and the OBJ / MTL writes.
What is stubbed: xatlas (returns this project's unwrapper output on the fixture mesh, stored in the fixture), dr.rasterize /
dr.interpolate (answered by nero_oracle_texmap.rasterize / interpolate), trimesh.load and open3d's mesh reader (the
fixture mesh), the ray tracer and the dataset split (unused by the export), torch.load (seeded, perturbed stage-II
parameters, as the material_* fixtures use) and cv2.imwrite (records its arrays).  TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(ROOT, 'tests', 'golden')
sys.path[:0] = [HERE, ROOT]

import nero_oracle as O  # noqa: E402
import nero_oracle_mat as OM  # noqa: E402
import nero_oracle_mesh as OMesh  # noqa: E402
import nero_oracle_texmap as OT  # noqa: E402

SHADER_CFG = {'human_lights': False, 'diffuse_sample_num': 16, 'specular_sample_num': 16}
SSAA = 2


def blob_mesh(n=20):
    """A bumpy blob from the oracle's marching cubes (many small triangles, several charts)."""
    ax = np.linspace(-1.0, 1.0, n)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    u = (np.linalg.norm(x * [1.0, 1.3, 0.8], axis=-1) - 0.7 + 0.12 * np.sin(4 * x[..., 0]) * np.cos(3 * x[..., 1])).astype(np.float32)
    v, t = OMesh.marching_cubes(u, 0.0)
    return (0.5 * v).astype(np.float32), t.astype(np.int32)


CASES = {
    'texmap_scene_32x32': (lambda: OM.test_scene(1), 32, 32, 11),
    'texmap_blob_40x64': (blob_mesh, 40, 64, 12),
}


def make_case(name, mesh_fn, h0, w0, pseed, seed=6033):
    import ref_shim
    from nero_b200 import params as PR
    from nero_b200 import texmap as TX
    verts, tris = mesh_fn()
    h, w = h0 * SSAA, w0 * SSAA
    vt, ft = TX.uv_atlas(verts, tris, w, h, 2 * SSAA)
    sd = O.perturb_params(PR.build_material_state_dict(SHADER_CFG, seed=seed), seed=pseed)
    rec = {'imwrite': {}, 'cvt': []}
    ref_shim.install()
    import nvdiffrast.torch as dr
    state = {}

    def rasterize(ctx, pos, tri, resolution):
        clip = pos[0].numpy()
        assert np.allclose((clip[:, :2] + 1) / 2, vt, atol=1e-6) and np.array_equal(tri.numpy(), ft)
        owner, count, bary = OT.rasterize(vt, ft, resolution[1], resolution[0])
        assert tuple(resolution) == (h, w) and count.max() <= 1
        state.update(owner=owner, bary=bary)
        rast = np.zeros((1, h, w, 4), np.float32)
        rast[0, ..., 3] = owner + 1
        return torch.from_numpy(rast), None

    def interpolate(attr, rast, faces):
        out = OT.interpolate(attr[0].numpy(), faces.numpy(), state['owner'], state['bary'])
        return torch.from_numpy(out[None]), None
    dr.rasterize, dr.interpolate = rasterize, interpolate
    dr.RasterizeGLContext = lambda *a, **k: None

    class Atlas:
        def add_mesh(self, v, f):
            assert np.array_equal(v, verts) and np.array_equal(f, tris)

        def generate(self, chart_options=None, pack_options=None):
            assert chart_options.max_iterations == 0

        def __getitem__(self, i):
            return np.arange(vt.shape[0]), ft.astype(np.uint32), vt
    import xatlas
    xatlas.Atlas = Atlas
    xatlas.ChartOptions = lambda: types.SimpleNamespace(max_iterations=4)
    xatlas.PackOptions = lambda: types.SimpleNamespace()
    import trimesh
    trimesh.load = lambda *a, **k: types.SimpleNamespace(vertices=verts.astype(np.float64), faces=tris.astype(np.int64))
    import open3d
    open3d.io = types.SimpleNamespace(read_triangle_mesh=lambda p: types.SimpleNamespace(vertices=verts, triangles=tris))
    import raytracing
    raytracing.RayTracer = lambda *a, **k: None
    import network.renderer as NR
    NR.parse_database_name = lambda name: None
    NR.get_database_split = lambda db, split: ([0], [1])
    sys.modules.pop('extract_materials_texture_map', None)
    import extract_materials_texture_map as EX
    EX.load_cfg = lambda path: {'name': 'fixture', 'mesh': 'fixture.ply', 'database_name': 'syn/fixture', 'shader_cfg': dict(SHADER_CFG)}
    EX.flags = types.SimpleNamespace(cfg='fixture.yaml')
    EX.torch.load = lambda path, *a, **k: {'step': 1, 'network_state_dict': sd}
    real_nn = EX.NearestNeighbors

    class NN:
        def __init__(self, **kw):
            self.nn = real_nn(**kw)

        def fit(self, x):
            rec['search'] = np.asarray(x).copy()
            self.nn.fit(x)
            return self

        def kneighbors(self, q):
            d, idx = self.nn.kneighbors(q)
            rec['inpaint'], rec['idx'] = np.asarray(q).copy(), idx.copy()
            return d, idx
    EX.NearestNeighbors = NN
    real_to = torch.Tensor.to
    torch.Tensor.to = lambda self, *a, **k: real_to(self, *[('cpu' if x == 'cuda' else x) for x in a],
                                                    **{kk: ('cpu' if vv == 'cuda' else vv) for kk, vv in k.items()})
    real_cvt = EX.cv2.cvtColor
    EX.cv2 = types.SimpleNamespace(cvtColor=lambda a, c: (rec['cvt'].append(a.copy()), real_cvt(a, c))[1], resize=EX.cv2.resize,
                                   COLOR_RGB2BGR=EX.cv2.COLOR_RGB2BGR, COLOR_GRAY2BGR=EX.cv2.COLOR_GRAY2BGR,
                                   INTER_LINEAR=EX.cv2.INTER_LINEAR,
                                   imwrite=lambda p, a: rec['imwrite'].__setitem__(os.path.basename(p), a.copy()))
    with tempfile.TemporaryDirectory() as tmp:
        out_dir = os.path.join(tmp, 'n2m_test')
        with ref_shim._cwd(ref_shim.REFERENCE_ROOT):     # assets/bsdf_256_256.bin is CWD-relative (field.py:510)
            torch.manual_seed(seed)
            xyzs, mask = EX.texture_mapper(path=out_dir, h0=h0, w0=w0)
        obj = open(os.path.join(out_dir, 'mesh_0.obj')).read()
        mtl = open(os.path.join(out_dir, 'mesh_0.mtl')).read()
    mask = mask.numpy().reshape(h, w)
    after = np.concatenate([rec['cvt'][0], rec['cvt'][1][..., None], rec['cvt'][2][..., None]], -1)
    inp = rec['inpaint'].astype(np.int64)
    before = after.copy()
    before[inp[:, 0], inp[:, 1]] = 0          # the inpainted texels were uncovered: encoded zeros before the copy
    src = rec['search'][rec['idx'][:, 0]].astype(np.int64)
    out = {'verts': verts, 'tris': tris, 'vt': vt, 'ft': ft, 'hw0': np.asarray([h0, w0]), 'ssaa': np.int64(SSAA), 'seed': np.int64(seed),
           'pseed': np.int64(pseed), 'xyzs': xyzs.numpy(), 'mask': mask, 'img_before': before, 'img_after': after,
           'inpaint_texels': inp[:, 0] * w + inp[:, 1], 'inpaint_src': src[:, 0] * w + src[:, 1],
           'feat0': rec['imwrite']['feat0_0.jpg'], 'feat1': rec['imwrite']['feat1_0.jpg'], 'feat2': rec['imwrite']['feat2_0.jpg'],
           'obj': np.asarray(obj), 'mtl': np.asarray(mtl)}
    np.savez_compressed(os.path.join(GOLD, name + '.npz'), **out)
    print(name, 'saved:', int(mask.sum()), 'covered texels,', inp.shape[0], 'inpainted,', {k: np.shape(v) for k, v in out.items()})


def main(ref):
    os.environ['NERO_REFERENCE_ROOT'] = ref
    import ref_shim
    ref_shim.REFERENCE_ROOT = ref
    for name, (mesh_fn, h0, w0, pseed) in CASES.items():
        make_case(name, mesh_fn, h0, w0, pseed)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
