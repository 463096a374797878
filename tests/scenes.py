"""Test-side scene helpers: everything of claymore_b200.scenes plus the oracle builders (tests only)."""
import hashlib
import os

import numpy as np

from claymore_b200.scenes import *  # noqa: F401,F403
from claymore_b200.scenes import material_parameters
from claymore_b200 import scenes as _pkg

J_FLUID, FIXED_COROTATED, SAND, NACC = 0, 1, 2, 3


def apply_material(sim, model_id, material, dx, is_oracle):
    """Engine: keyword `model`; oracle binding: model id first."""
    name, args = material_parameters(material, dx)
    if is_oracle:
        getattr(sim, name)(model_id, *args)
    else:
        getattr(sim, name)(*args, model=model_id)


def build_oracle(ob, scene, dt=1e-4, max_blocks=4000, max_ppc=128, threads=1, cfl=0.5, sim_class=None):
    """The oracle simulator of a scene, set up: an ob.OracleSim, or a sim_class such as collider_oracle_binding.ColliderOracleSim
    (boundaries)."""
    cfg = ob.make_config(domain_bits=scene["domain_bits"], max_ppc=max_ppc, cfl=cfl)
    sim = (sim_class or ob.OracleSim)(cfg, dt, max_blocks, threads=threads)
    dx = 1.0 / (1 << scene["domain_bits"])
    for m in scene["models"]:
        mid = sim.init_model(m["material"], m["pos"], m["v0"])
        apply_material(sim, mid, m["material"], dx, True)
    sim.initial_setup()
    return sim


def match_particles(a, b, tol):
    """Bijective nearest-neighbour match of two particle sets by position; returns index array into b."""
    from scipy.spatial import cKDTree
    d, idx = cKDTree(b[:, :3]).query(a[:, :3], k=1)
    assert d.max() <= tol, f"unmatched particle: nearest distance {d.max():.3e} > {tol:.3e}"
    assert len(np.unique(idx)) == len(a), "particle match is not a bijection"
    return idx


def load_ref_math_golden():
    """The reference's SVD / constitutive-model outputs on 4000 vectors (tests/golden/make_ref_math_golden.py), one dict."""
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    return {**np.load(os.path.join(d, "ref_math_golden_svd.npz")), **np.load(os.path.join(d, "ref_math_golden_stress.npz"))}


def key_digest(hashes):
    """SHA-256 of a set of block-key hashes (order-free): how the benchmark-scale fixtures store key sets."""
    return np.frombuffer(hashlib.sha256(np.sort(np.asarray(hashes, np.int64)).astype("<i8").tobytes()).digest(), np.uint8)
