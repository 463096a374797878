"""Scene / material front-end: the JSON schema of the reference's gmpm (Projects/GMPM/gmpm.cu:60-165,
Projects/GMPM/scenes/scene.json) mapped onto GmpmSimulator.

    {"simulation": {"gpuid", "fps", "frames", "default_dt"},
     "models": [{"type": "particles", "file": ..., "constitutive": "fixed_corotated"|"jfluid"|"nacc"|"sand",
                 "offset": [3], "span": [3], "velocity": [3], + material parameters}]}

     "collider": {"file": <prefix of <prefix>_sdf.bin / _grad_{0,1,2}.bin> | "box" | "sphere" | "plane",
                  "offset": [3], "span": [3], "normal": [3], "type": "sticky"|"slip"|"separate",
                  "friction", "velocity": [3], "omega": [3], "scale", "dsdt"}}

A "box" collider spans [offset, offset + span], a "sphere" has diameter min(span) at offset + span / 2, a "plane" passes
through offset and is solid behind `normal`.  The collider is the reference's SignedDistanceGrid (init_boundary,
Projects/MGSP/mgsp_benchmark.cuh:257-266); "velocity" is its trans_vel.

The reference only loads `.sdf` level sets (gmpm.cu:152, needs the absent Data submodule); here a model may also
name a synthetic generator: "file": "box" (span in cells of the lattice sampler) or "sphere" (span = diameter),
or a raw float32 xyz `.bin` cloud as used by mgsp.cu:11-17.
"""
import json
import os

import numpy as np

from . import levelset, samplers
from ._capi import Config, FIXED_COROTATED, J_FLUID, NACC, SAND
from .simulator import GmpmSimulator

CONSTITUTIVE = {"jfluid": J_FLUID, "fixed_corotated": FIXED_COROTATED, "sand": SAND, "nacc": NACC}


def _positions(model, cfg, base_dir):
    dx = cfg.dx
    offset = np.asarray(model.get("offset", [0, 0, 0]), dtype=np.float64)
    span = np.asarray(model.get("span", [1, 1, 1]), dtype=np.float64)
    kind = model.get("file", "box")
    if kind == "box":
        lo = np.round(offset / dx).astype(int)
        hi = np.round((offset + span) / dx).astype(int)
        return samplers.uniform_box(dx, lo, hi)
    if kind == "sphere":
        return samplers.sphere(dx, offset + span / 2, float(span.min()) / 2)
    path = kind if os.path.isabs(kind) else os.path.join(base_dir, kind)
    if path.endswith(".bin"):
        return np.fromfile(path, dtype=np.float32).reshape(-1, 3)
    if path.endswith(".npy"):
        return np.load(path).astype(np.float32).reshape(-1, 3)
    raise ValueError(f"unsupported model file {kind!r} (the reference's .sdf sampler is outside the hot path)")


def _collider(sim, c, cfg, base_dir):
    kind = c.get("file", "box")
    offset = np.asarray(c.get("offset", [0, 0, 0]), dtype=np.float64)
    span = np.asarray(c.get("span", [1, 1, 1]), dtype=np.float64)
    if kind == "box":
        sdf, grad = levelset.box(cfg, offset, offset + span)
    elif kind == "sphere":
        sdf, grad = levelset.sphere(cfg, offset + span / 2, float(span.min()) / 2)
    elif kind == "plane":
        sdf, grad = levelset.plane(cfg, offset, c.get("normal", [0, 1, 0]))
    else:
        sdf, grad = levelset.load(cfg, kind if os.path.isabs(kind) else os.path.join(base_dir, kind))
    sim.set_collider(sdf, grad, type=c.get("type", "sticky"), friction=c.get("friction", 0.3), trans_vel=c.get("velocity", [0, 0, 0]),
                     omega=c.get("omega", [0, 0, 0]), scale=c.get("scale", 1.0), dsdt=c.get("dsdt", 0.0))


def parse_scene(path_or_dict, config=None, max_blocks=10000, **sim_kwargs):
    """parse_scene (gmpm.cu:60-165): returns an initialised GmpmSimulator with every model registered."""
    if isinstance(path_or_dict, dict):
        doc, base = path_or_dict, os.getcwd()
    else:
        with open(path_or_dict) as f:
            doc = json.load(f)
        base = os.path.dirname(os.path.abspath(path_or_dict))
    cfg = config if config is not None else Config()
    s = doc.get("simulation", {})
    sim = GmpmSimulator(gpu=s.get("gpuid", 0), dt=s.get("default_dt", GmpmSimulator.DEFAULT_DT), fps=s.get("fps", GmpmSimulator.DEFAULT_FPS),
                        frames=s.get("frames", GmpmSimulator.DEFAULT_FRAMES), config=cfg, max_blocks=max_blocks, **sim_kwargs)
    for model in doc.get("models", []):
        if model.get("type", "particles") != "particles":
            continue
        c = model["constitutive"]
        if c not in CONSTITUTIVE:
            raise ValueError(f"unknown constitutive model {c!r}")
        pos = _positions(model, cfg, base)
        mid = sim.init_model(CONSTITUTIVE[c], pos, model.get("velocity", [0, 0, 0]))
        # material parameters exactly as gmpm.cu:108-150 forwards them
        if c == "jfluid":
            sim.update_j_fluid_parameters(model["rho"], model["volume"], model["bulk_modulus"], model["gamma"], model["viscosity"], model=mid)
        elif c == "fixed_corotated":
            sim.update_fr_parameters(model["rho"], model["volume"], model["youngs_modulus"], model["poisson_ratio"], model=mid)
        elif c == "nacc":
            sim.update_nacc_parameters(model["rho"], model["volume"], model["youngs_modulus"], model["poisson_ratio"], model["beta"], model["xi"], model=mid)
        elif c == "sand" and "youngs_modulus" in model:  # the reference leaves sand at its defaults (gmpm.cu:134-135)
            sim.update_sand_parameters(model["rho"], model["volume"], model["youngs_modulus"], model["poisson_ratio"], model=mid)
    if "collider" in doc:
        _collider(sim, doc["collider"], cfg, base)
    return sim
