"""Generate tests/golden/relight_poses.npz from the UNMODIFIED reference's camera algebra (needs a checkout of the reference
repository; no Blender).

    python oracle/make_golden_relight.py <path to the reference checkout>

Runs the reference's generate_relghting_poses and set_camera_by_pose (blender_backend/blender_utils.py:48-68, 101-116) with
`bpy` stubbed and a stand-in camera object, then turns the camera's Blender location and rotation quaternion (camera to
world, Blender camera axes x right, y up, z backwards) into world -> camera [R | t] with OpenCV axes, the form
nero_b200.relight.relight_poses returns.  TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
CONFIGS = [(7, 0.0, 45.0, 3.0), (5, 30.0, 20.0, 2.5), (4, -60.0, 70.0, 1.5)]


class _Camera:
    def __init__(self):
        self.location = [0.0, 0.0, 0.0]
        self.rotation_quaternion = [1.0, 0.0, 0.0, 0.0]
        self.rotation_mode = 'XYZ'


def quat_to_matrix(q):
    w, x, y, z = q
    return np.asarray([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                       [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                       [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def main(ref):
    sys.modules['bpy'] = types.ModuleType('bpy')
    sys.path.insert(0, ref)
    from blender_backend.blender_utils import generate_relghting_poses, set_camera_by_pose
    out = {}
    for c, (num, az, el, dist) in enumerate(CONFIGS):
        poses = generate_relghting_poses(num, az, el, dist)
        res = []
        for k in range(num):
            cam = _Camera()
            set_camera_by_pose(cam, poses[k])
            c2w_gl = quat_to_matrix(np.asarray(cam.rotation_quaternion, np.float64))
            R = np.diag([1.0, -1.0, -1.0]) @ c2w_gl.T          # world -> camera, OpenCV axes
            t = -R @ np.asarray(cam.location, np.float64)
            res.append(np.concatenate([R, t[:, None]], 1))
        out[f'config{c}'] = np.asarray([num, az, el, dist], np.float64)
        out[f'poses{c}'] = np.stack(res)
    np.savez_compressed(os.path.join(GOLD, 'relight_poses.npz'), **out)
    print('relight_poses saved', {k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main(sys.argv[1])
