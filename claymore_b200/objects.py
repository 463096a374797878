"""Analytic collision objects (GmpmSimulator.set_collision_objects, DESIGN.md section 2.9).

Each constructor returns a cb200_collision_object.  The shape is written in the collider's material space, which is world space
for a static object, so a shape is placed in world coordinates at t = 0 and moves exactly as a level-set collider with the same
motion parameters would.  The keyword arguments and their defaults are GmpmSimulator.set_collider's:
type ("sticky" / "slip" / "separate" or CB200_*), friction, trans, trans_vel, omega, rot (3x3, row i, column j = rot_mat(i, j)),
scale, dsdt.

objects.levelset places an SDFGen level set (claymore_b200.sdf.LevelSet) as an obstacle (DESIGN.md section 2.11): the simulator
registers its lattice on first use and writes the registry index into the object it passes on.

objects.track(keys, interp, periodic) is a motion track (DESIGN.md section 2.14): keyframed poses of the object's pivot and rotation
that the grid update evaluates at each sub-step's time.  Every constructor takes it as track=; the object then places its shape with
R(t) = Q(t) rot about the pivot c(t) (x = R(t)^T (p - c(t)) scale + trans) and moves rigidly, so trans_vel, omega and dsdt must be 0.
"""
import math

import numpy as np

from ._capi import (MAX_COLLISION_LEVELSETS, MAX_COLLISION_OBJECTS, MAX_TRACK_KEYS, SEPARATE, SHAPE_BOX, SHAPE_CYLINDER, SHAPE_LEVELSET,
                    SHAPE_PLANE, SHAPE_SPHERE, SLIP, STICKY, TRACK_LINEAR, TRACK_PERIODIC, TRACK_SMOOTH, CollisionObject, TrackKey)

BOUNDARY_TYPES = {"sticky": STICKY, "slip": SLIP, "separate": SEPARATE}
SHAPES = {"plane": SHAPE_PLANE, "box": SHAPE_BOX, "sphere": SHAPE_SPHERE, "cylinder": SHAPE_CYLINDER}


def _vec(v, n=3, what="vector"):
    a = np.asarray(v, np.float64).reshape(-1)
    if a.size != n:
        raise ValueError(f"{what} must have {n} components, not {a.size}")
    return [float(x) for x in a]


def _make(shape, a, b, type="sticky", friction=0.3, trans=(0.0, 0.0, 0.0), trans_vel=(0.0, 0.0, 0.0), omega=(0.0, 0.0, 0.0), rot=None,
          scale=1.0, dsdt=0.0, track=None):
    o = CollisionObject()
    o.shape = shape
    if isinstance(type, str):
        if type not in BOUNDARY_TYPES:
            raise ValueError(f"unknown boundary type {type!r} (known: {', '.join(BOUNDARY_TYPES)})")
        o.type = BOUNDARY_TYPES[type]
    else:
        o.type = int(type)
    o.friction = float(friction)
    o.a[:], o.b[:] = a, b
    o.rot_mat[:] = _vec(np.eye(3) if rot is None else rot, 9, "rot")
    o.trans[:], o.trans_vel[:], o.omega[:] = _vec(trans, what="trans"), _vec(trans_vel, what="trans_vel"), _vec(omega, what="omega")
    o.scale, o.dsdt = float(scale), float(dsdt)
    validate(o)
    if track is not None:
        if not isinstance(track, Track):
            raise ValueError("track must come from objects.track")
        if any(o.trans_vel) or any(o.omega) or o.dsdt != 0.0:
            raise ValueError("a tracked object must have trans_vel = omega = 0 and dsdt = 0: the track moves it")
        o.track = track
    return o


# ---- motion tracks (DESIGN.md section 2.14) -----------------------------------------------------------------------------------
INTERP = {"linear": TRACK_LINEAR, "smooth": TRACK_SMOOTH}


class Track:
    """A validated motion track: keys (a ctypes array of cb200_track_key), n and flags (CB200_TRACK_*), as
    GmpmSimulator.set_object_track passes them on."""

    def __init__(self, keys, flags):
        self.keys, self.n, self.flags = keys, len(keys), flags


def quaternion(rotation):
    """The unit quaternion (w, x, y, z) of a rotation given as a quaternion (4 values) or a 3x3 rotation matrix (row i, column j), in
    double; a zero quaternion or a matrix that is not a rotation raises ValueError."""
    r = np.asarray(rotation, np.float64)
    if r.shape == (4,):
        if not np.isfinite(r).all():
            raise ValueError("every value of a track key must be finite")
        n = np.linalg.norm(r)
        if not n > 0:
            raise ValueError("a track key's quaternion must not be zero")
        return r / n
    if r.shape != (3, 3):
        raise ValueError(f"a rotation is a quaternion (w, x, y, z) or a 3x3 matrix, not shape {r.shape}")
    if not np.isfinite(r).all():
        raise ValueError("every value of a track key must be finite")
    if not (np.allclose(r @ r.T, np.eye(3), atol=1e-5) and np.linalg.det(r) > 0):
        raise ValueError("a track key's matrix must be a rotation")
    # the largest of w, x, y, z first (Shepperd), then the rest from the off-diagonal terms
    tr = np.trace(r)
    cand = [tr, r[0, 0], r[1, 1], r[2, 2]]
    i = int(np.argmax(cand))
    if i == 0:
        w = np.sqrt(1.0 + tr) / 2
        q = [w, (r[2, 1] - r[1, 2]) / (4 * w), (r[0, 2] - r[2, 0]) / (4 * w), (r[1, 0] - r[0, 1]) / (4 * w)]
    else:
        a, b, c = [(0, 1, 2), (1, 2, 0), (2, 0, 1)][i - 1]
        v = np.sqrt(1.0 + r[a, a] - r[b, b] - r[c, c]) / 2
        q = np.zeros(4)
        q[0] = (r[c, b] - r[b, c]) / (4 * v)
        q[1 + a] = v
        q[1 + b] = (r[b, a] + r[a, b]) / (4 * v)
        q[1 + c] = (r[c, a] + r[a, c]) / (4 * v)
    q = np.asarray(q, np.float64)
    return q / np.linalg.norm(q)


def track(keys, interp="linear", periodic=False):
    """A motion track from keys [(t, position, rotation)], rotation a quaternion (w, x, y, z) or a 3x3 rotation matrix: the checks of
    cb200_track_prepare as ValueError (1 to MAX_TRACK_KEYS keys with strictly increasing t, finite values, no zero quaternion, no two
    neighbouring rotations 180 degrees apart, a periodic track's last pose equal to its first, quaternions up to sign).  interp:
    "linear" (piecewise linear positions) or "smooth" (cubic Hermite); every segment's rotation is a slerp."""
    if interp not in INTERP:
        raise ValueError(f"unknown interpolation {interp!r} (known: {', '.join(INTERP)})")
    keys = list(keys)
    if not 1 <= len(keys) <= MAX_TRACK_KEYS:
        raise ValueError(f"a track has 1 to {MAX_TRACK_KEYS} keys, not {len(keys)}")
    if periodic and len(keys) < 2:
        raise ValueError("a periodic track needs at least 2 keys")
    arr = (TrackKey * len(keys))()
    qs = []
    for k, key in enumerate(keys):
        if len(key) != 3:
            raise ValueError("a track key is (t, position, rotation)")
        t, pos, rot = key
        pos = _vec(pos, what="position")
        if not (math.isfinite(float(t)) and all(math.isfinite(v) for v in pos)):
            raise ValueError("every value of a track key must be finite")
        q = quaternion(rot)
        arr[k].t, arr[k].pos[:], arr[k].rot[:] = float(t), pos, [float(v) for v in q]
        if k > 0 and not arr[k].t > arr[k - 1].t:
            raise ValueError(f"track key times must increase strictly (as float32): {arr[k - 1].t} then {arr[k].t}")
        qs.append(np.asarray(list(arr[k].rot), np.float64))
    for k in range(1, len(qs)):
        a = qs[k - 1] / np.linalg.norm(qs[k - 1])
        b = qs[k] / np.linalg.norm(qs[k])
        if float(a @ b) == 0.0:
            raise ValueError(f"track keys {k - 1} and {k} are 180 degrees apart: the rotation between them is ambiguous")
        if float(a @ b) < 0.0:
            qs[k] = -qs[k]
    if periodic:
        f32 = lambda v: np.asarray(v, np.float64) / np.linalg.norm(np.asarray(v, np.float64))  # noqa: E731
        first, last = arr[0], arr[len(keys) - 1]
        q0, q1 = f32(list(first.rot)).astype(np.float32), f32(list(last.rot)).astype(np.float32)
        if list(first.pos) != list(last.pos) or not (np.array_equal(q0, q1) or np.array_equal(q0, -q1)):
            raise ValueError("a periodic track's last pose must equal its first")
    return Track(arr, INTERP[interp] | (TRACK_PERIODIC if periodic else 0))


def plane(point, normal, **motion):
    """Half-space solid where (x - point) . normal <= 0; the normal is made unit length in double (as levelset.plane does)."""
    n = np.asarray(_vec(normal, what="normal"))
    ln = np.linalg.norm(n)
    if not ln > 0:
        raise ValueError("a plane's normal must not be zero")
    return _make(SHAPE_PLANE, _vec(point, what="point"), [float(v) for v in n / ln], **motion)


def box(lo, hi, **motion):
    """Axis-aligned box [lo, hi] (in material space)."""
    return _make(SHAPE_BOX, _vec(lo, what="lo"), _vec(hi, what="hi"), **motion)


def sphere(centre, radius, **motion):
    return _make(SHAPE_SPHERE, _vec(centre, what="centre"), [float(radius), 0.0, 0.0], **motion)


def cylinder(centre, radius, half_height, **motion):
    """Capped cylinder with its axis along material-space y through centre (orient it with rot)."""
    return _make(SHAPE_CYLINDER, _vec(centre, what="centre"), [float(radius), float(half_height), 0.0], **motion)


def levelset(ls, offset, span, **motion):
    """The level set `ls` (claymore_b200.sdf.LevelSet) as an obstacle fitted into [offset, offset + span] with the sampler's uniform
    fit (sdf.node_box): node (0, 0, 0) at offset, node spacing its cell size.  Solid where phi <= 0.  The box may extend past the
    domain.  b[1], the registry index, is written by GmpmSimulator when it registers `ls`."""
    from . import sdf
    if not min(sdf._vec3(span)) > 0:
        raise ValueError(f"span {sdf._vec3(span)} must be positive")
    c, lo, _ = sdf.node_box(ls, offset, span)
    o = _make(SHAPE_LEVELSET, lo, [c, 0.0, 0.0], **motion)
    o.levelset = ls
    return o


def validate(o, levelsets=MAX_COLLISION_LEVELSETS):
    """The checks of cb200_sim_set_collision_objects, as ValueError: unknown shape or type, scale 0, a non-finite value, a zero
    plane normal, lo > hi, a radius or half height <= 0, a level set's spacing <= 0 or an index that is not an integer in
    [0, levelsets) (the registry's size)."""
    if o.shape not in SHAPES.values() and o.shape != SHAPE_LEVELSET:
        raise ValueError(f"unknown shape {o.shape}")
    if o.type not in BOUNDARY_TYPES.values():
        raise ValueError(f"unknown boundary type {o.type}")
    vals = [o.friction, o.dsdt, o.scale, *o.a, *o.b, *o.rot_mat, *o.trans, *o.trans_vel, *o.omega]
    if not all(math.isfinite(v) for v in vals):
        raise ValueError("every value of a collision object must be finite")
    if o.scale == 0.0:
        raise ValueError("scale must not be 0")
    if o.shape == SHAPE_PLANE and not any(o.b):
        raise ValueError("a plane's normal must not be zero")
    if o.shape == SHAPE_BOX and any(lo > hi for lo, hi in zip(o.a, o.b)):
        raise ValueError(f"a box needs lo <= hi, not {list(o.a)} > {list(o.b)}")
    if o.shape in (SHAPE_SPHERE, SHAPE_CYLINDER) and not o.b[0] > 0:
        raise ValueError(f"a radius must be positive, not {o.b[0]}")
    if o.shape == SHAPE_CYLINDER and not o.b[1] > 0:
        raise ValueError(f"a half height must be positive, not {o.b[1]}")
    if o.shape == SHAPE_LEVELSET:
        if not o.b[0] > 0:
            raise ValueError(f"a level set's node spacing must be positive, not {o.b[0]}")
        if not (o.b[1] == int(o.b[1]) and 0 <= o.b[1] < levelsets):
            raise ValueError(f"a level set's index must be an integer in [0, {levelsets}), not {o.b[1]}")
    return o


def array(objs, levelsets=MAX_COLLISION_LEVELSETS):
    """ctypes array of the validated objects (at most MAX_COLLISION_OBJECTS; level-set indices below `levelsets`)."""
    objs = list(objs)
    if len(objs) > MAX_COLLISION_OBJECTS:
        raise ValueError(f"at most {MAX_COLLISION_OBJECTS} collision objects, not {len(objs)}")
    for o in objs:
        validate(o, levelsets)
    return (CollisionObject * max(len(objs), 1))(*objs)
