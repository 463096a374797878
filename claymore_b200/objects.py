"""Analytic collision objects (GmpmSimulator.set_collision_objects, DESIGN.md section 2.9).

Each constructor returns a cb200_collision_object.  The shape is written in the collider's material space, which is world space
for a static object, so a shape is placed in world coordinates at t = 0 and moves exactly as a level-set collider with the same
motion parameters would.  The keyword arguments and their defaults are GmpmSimulator.set_collider's:
type ("sticky" / "slip" / "separate" or CB200_*), friction, trans, trans_vel, omega, rot (3x3, row i, column j = rot_mat(i, j)),
scale, dsdt.

objects.levelset places an SDFGen level set (claymore_b200.sdf.LevelSet) as an obstacle (DESIGN.md section 2.11): the simulator
registers its lattice on first use and writes the registry index into the object it passes on.
"""
import math

import numpy as np

from ._capi import (MAX_COLLISION_LEVELSETS, MAX_COLLISION_OBJECTS, SEPARATE, SHAPE_BOX, SHAPE_CYLINDER, SHAPE_LEVELSET, SHAPE_PLANE,
                    SHAPE_SPHERE, SLIP, STICKY, CollisionObject)

BOUNDARY_TYPES = {"sticky": STICKY, "slip": SLIP, "separate": SEPARATE}
SHAPES = {"plane": SHAPE_PLANE, "box": SHAPE_BOX, "sphere": SHAPE_SPHERE, "cylinder": SHAPE_CYLINDER}


def _vec(v, n=3, what="vector"):
    a = np.asarray(v, np.float64).reshape(-1)
    if a.size != n:
        raise ValueError(f"{what} must have {n} components, not {a.size}")
    return [float(x) for x in a]


def _make(shape, a, b, type="sticky", friction=0.3, trans=(0.0, 0.0, 0.0), trans_vel=(0.0, 0.0, 0.0), omega=(0.0, 0.0, 0.0), rot=None,
          scale=1.0, dsdt=0.0):
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
    return o


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
