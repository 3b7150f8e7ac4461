"""Seeded keyframes for the occupancy-grid tests: small scenes that hit each of the grid_mapping tool's quirks, and keyframe point
sets in the dense map's format.  A scene is (cfg, keyframes): cfg holds GridMap's keyword arguments, keyframes is a list of
(R, P, points float32 (n, 3))."""
import math

import numpy as np

import dm_scenes


def _pts(a):
    return np.asarray(a, np.float32).reshape(-1, 3)


def ring(rng, n, rmin, rmax, z):
    """n camera-frame points (ric = I) at horizontal distance [rmin, rmax] around the body, height z (array or scalar)."""
    a = rng.uniform(-math.pi, math.pi, n)
    r = rng.uniform(rmin, rmax, n)
    return _pts(np.stack([r * np.cos(a), r * np.sin(a), np.broadcast_to(z, (n,))], 1))


def band_edge_z():
    """float32 heights h and body heights Pz with h + Pz == 0.1 and == 0.5 exactly in double, and the neighbours just outside."""
    out = []
    for target in (0.1, 0.5):
        for h in (np.float32(0.25), np.float32(0.3), np.float32(0.7)):
            pz = target - float(h)
            if float(h) + pz == target:
                out.append((h, pz, True))
                q = pz
                while float(h) + q == target:
                    q = math.nextafter(q, -math.inf if target == 0.1 else math.inf)
                out.append((h, q, False))
    return out


def quirk_scenes():
    rng = np.random.default_rng(11)
    eye = np.eye(3)
    small = dict(size_x=60, size_y=40, init_x=30, init_y=20, cell_size=0.05)
    scenes = []
    # a body at exactly (-1, -1): every ray skips its first cell; the grid covers negative coordinates
    scenes.append(("body_at_minus_one", dict(small, init_x=45, init_y=35),
                   [(eye, np.array([-1.0, -1.0, 0.0]), ring(rng, 40, 0.2, 1.2, 0.3))]))
    # points straight above / below the body (dx = dy = 0) among ordinary ones
    pts = np.concatenate([_pts([[0, 0, 0.3], [0, 0, 0.45], [0, 0, 0.2]]), ring(rng, 20, 0.1, 0.8, 0.3)])
    scenes.append(("point_above_body", small, [(eye, np.array([0.2, -0.1, 0.0]), pts), (eye, np.array([0.0, 0.0, 0.0]), pts)]))
    # world z exactly 0.1 and 0.5 (kept) and just outside (dropped)
    kfs = []
    for h, pz, _ in band_edge_z():
        kfs.append((eye, np.array([0.03, 0.02, pz]), _pts(np.stack([rng.uniform(-0.9, 0.9, 12), rng.uniform(-0.9, 0.9, 12), np.full(12, h)], 1))))
    scenes.append(("band_edges", small, kfs))
    # rays leaving the grid on each side (and corners); negative coordinates
    scenes.append(("leaving_the_grid", dict(size_x=24, size_y=18, init_x=12, init_y=9, cell_size=0.05),
                   [(eye, np.array([0.1, -0.05, 0.0]), ring(rng, 60, 0.3, 3.0, 0.3)),
                    (dm_scenes.rot(0, 0, 0.7), np.array([-0.4, -0.3, 0.1]), ring(rng, 60, 0.3, 3.0, 0.2))]))
    # the same points again and again: free runs into bel = 2^-52, occupied runs into 1 - 2^-53, prior steps at the ray end
    rep = np.repeat(ring(rng, 6, 0.3, 0.7, 0.3), 50, axis=0)
    scenes.append(("fixed_points", small, [(eye, np.array([0.0, 0.0, 0.0]), rep)] * 3))
    # p_occ = 0.9: occupied cells reach bel == 1 exactly and stay there; p_free = 0.2 reaches 0
    scenes.append(("absorbing", dict(small, p_occ=0.9, p_free=0.2), [(eye, np.array([0.01, 0.0, 0.0]), rep)] * 2))
    # a general pose and extrinsic, cell size not a power of two, steps repeating a cell
    ric = dm_scenes.rot(0.02, -0.01, 0.3)
    scenes.append(("general", dict(size_x=50, size_y=50, init_x=20, init_y=30, cell_size=0.07, p_occ=0.7, p_free=0.35, p_prior=0.45,
                                   ric=ric, tic=np.array([0.02, -0.03, 0.05])),
                   [(dm_scenes.rot(0.03, 0.02, 0.1 * k), np.array([0.05 * k, -0.02 * k, 0.01]),
                     _pts(np.stack([rng.uniform(-2, 2, 80), rng.uniform(-2, 2, 80), rng.uniform(0.0, 0.6, 80)], 1))) for k in range(4)]))
    return scenes


def keyframe_points(k, n=3000):
    """Keyframe k's points in the dense map's row format (n, 6): camera-frame x y z at depths 0.3 .. 7 m, then r g b."""
    rng = np.random.default_rng(1000 + k)
    d = rng.uniform(0.3, 7.0, n)
    u, v = rng.uniform(-0.7, 0.7, n), rng.uniform(-0.5, 0.5, n)
    out = np.zeros((n, 6), np.float32)
    out[:, 0], out[:, 1], out[:, 2] = u * d, v * d, d
    out[:, 3:] = rng.integers(0, 256, (n, 3))
    return out


def camera_to_body():
    """A forward-looking camera: camera z along body x, camera y along -body z (the tool's hard-coded extrinsic's shape)."""
    return np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]]), np.array([0.04, 0.03, 0.3])


def body_pose(k):
    """A ground vehicle's body pose: yaw and a small pitch / roll, position wandering around the origin at z ~ 0."""
    t = 0.05 * k
    return dm_scenes.rot(0.02 * math.sin(t), 0.03 * math.sin(0.7 * t), 0.4 * t), np.array([3.0 * math.sin(t), 2.0 * math.sin(0.5 * t), 0.02 * math.sin(t)])
