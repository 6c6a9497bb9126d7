"""Procedural meshes in mm with known rotational symmetry groups, for the symmetry finder's tests.

EXPECTED[name] = (number of discrete symmetries, continuous axis or None) as find_symmetries reports them for the mesh as
built; placed() moves a mesh off the origin and rotates it, which moves its axes with it."""
import math

import numpy as np

from sam6d_b200 import meshio

FACE_COLOURS = np.array([[230, 30, 30], [30, 230, 30], [30, 30, 230], [230, 230, 30], [230, 30, 230], [30, 230, 230]], np.uint8)


def _mesh(verts, faces, colors=None):
    return meshio.Mesh(vertices=np.asarray(verts, np.float32), faces=np.asarray(faces, np.int64),
                       colors=None if colors is None else np.asarray(colors, np.uint8))


def box(sx, sy, sz, face_colors=None):
    """an axis-aligned box centred at the origin, each face with its own 4 vertices (face_colors (6,3) u8: -x, +x, -y, +y, -z, +z)"""
    verts, faces, cols = [], [], []
    h = np.array([sx, sy, sz], np.float64) / 2.0
    for axis in range(3):
        for side, sgn in enumerate((-1.0, 1.0)):
            u, v = [(axis + 1) % 3, (axis + 2) % 3]
            quad = []
            for a, b in ((-1, -1), (1, -1), (1, 1), (-1, 1)):
                p = np.zeros(3)
                p[axis], p[u], p[v] = sgn * h[axis], a * h[u], b * h[v]
                quad.append(p)
            o = len(verts)
            verts += quad
            faces += [[o, o + 1, o + 2], [o, o + 2, o + 3]] if sgn > 0 else [[o, o + 2, o + 1], [o, o + 3, o + 2]]
            if face_colors is not None:
                cols += [face_colors[2 * axis + side]] * 4
    return _mesh(verts, faces, cols if face_colors is not None else None)


def prism(n, r, h):
    """a regular n-gon prism about z (a vertex on +x), circumradius r, height h, closed by two fans"""
    ang = 2.0 * math.pi * np.arange(n) / n
    ring = np.stack([r * np.cos(ang), r * np.sin(ang)], axis=1)
    verts = [[x, y, -h / 2] for x, y in ring] + [[x, y, h / 2] for x, y in ring] + [[0, 0, -h / 2], [0, 0, h / 2]]
    faces = []
    for i in range(n):
        j = (i + 1) % n
        faces += [[i, j, n + j], [i, n + j, n + i], [2 * n, j, i], [2 * n + 1, n + i, n + j]]
    return _mesh(verts, faces)


def cone(n, r, h):
    """a cone about z: base circle (n segments) of radius r at z = -h/3, apex at z = 2h/3, closed by a fan"""
    ang = 2.0 * math.pi * np.arange(n) / n
    verts = [[r * math.cos(a), r * math.sin(a), -h / 3] for a in ang] + [[0, 0, 2 * h / 3], [0, 0, -h / 3]]
    faces = []
    for i in range(n):
        j = (i + 1) % n
        faces += [[i, j, n], [n + 1, j, i]]
    return _mesh(verts, faces)


def blob(r=50.0, n_lat=40, n_lon=80):
    """a closed lumpy sphere with no rotational symmetry"""
    verts = [[0, 0, r * 1.0]]
    for i in range(1, n_lat):
        th = math.pi * i / n_lat
        for k in range(n_lon):
            ph = 2.0 * math.pi * k / n_lon
            d = np.array([math.sin(th) * math.cos(ph), math.sin(th) * math.sin(ph), math.cos(th)])
            x, y, z = d
            s = 1.0 + 0.3 * x + 0.2 * y * y + 0.25 * x * z + 0.3 * y * z * z + 0.15 * x * y + 0.1 * z
            verts.append(list(r * s * d))
    verts.append([0, 0, -r * 0.9])
    faces, last = [], len(verts) - 1
    ring = lambda i, k: 1 + (i - 1) * n_lon + (k % n_lon)
    for k in range(n_lon):
        faces.append([0, ring(1, k), ring(1, k + 1)])
        faces.append([last, ring(n_lat - 1, k + 1), ring(n_lat - 1, k)])
    for i in range(1, n_lat - 1):
        for k in range(n_lon):
            a, b, c, d = ring(i, k), ring(i, k + 1), ring(i + 1, k + 1), ring(i + 1, k)
            faces += [[a, d, c], [a, c, b]]
    return _mesh(verts, faces)


def build(name):
    if name == "blob":
        return blob()
    if name == "box3":
        return box(100.0, 70.0, 40.0)
    if name == "square_prism":
        return box(60.0, 60.0, 110.0)
    if name == "hex_prism":
        return prism(6, 40.0, 70.0)
    if name == "cube":
        return box(80.0, 80.0, 80.0)
    if name == "cube_colours":
        return box(80.0, 80.0, 80.0, FACE_COLOURS)
    if name == "cube_opposite":
        return box(80.0, 80.0, 80.0, FACE_COLOURS[[0, 0, 1, 1, 2, 2]])
    if name == "cylinder":
        return prism(128, 35.0, 90.0)
    if name == "cone":
        return cone(128, 40.0, 90.0)
    raise KeyError(name)


EXPECTED = {"blob": (0, None), "box3": (3, None), "square_prism": (7, None), "hex_prism": (11, None), "cube": (23, None),
            "cube_colours": (0, None), "cube_opposite": (3, None), "cylinder": (1, (0.0, 0.0, 1.0)), "cone": (0, (0.0, 0.0, 1.0))}
NAMES = tuple(EXPECTED)


def placed(mesh, rot=None, shift=(30.0, -20.0, 55.0)):
    """the mesh rotated by rot (3,3) about the origin, then shifted by `shift` mm"""
    R = np.eye(3) if rot is None else np.asarray(rot, np.float64)
    v = np.asarray(mesh.vertices, np.float64) @ R.T + np.asarray(shift, np.float64)
    return meshio.Mesh(vertices=v.astype(np.float32), faces=mesh.faces, colors=mesh.colors)


def random_rotation(seed=3):
    from scipy.spatial.transform import Rotation
    return Rotation.random(random_state=seed).as_matrix()
