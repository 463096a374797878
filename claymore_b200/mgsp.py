"""MGSP host layer: static particle partition across one-process-per-GPU ranks (Projects/MGSP/mgsp.cu:34-96,
mgsp_benchmark.cuh:240-334 in the reference, where one process drives all GPUs with a worker thread each).

torch.distributed is used for plumbing only: rendezvous, the one-time all-gather of the 64-byte CUDA-IPC inbox handles,
barriers and the max-over-ranks of the timings.  The per-sub-step exchange (halo grid blocks, neighbour keys, max |v|^2)
is done by the library's kernels through peer memory; see csrc/mgsp.cuh.
"""
import numpy as np

from . import samplers
from ._capi import Config
from .simulator import GmpmSimulator


def partition_scene(scene, rank, world, axis=0):
    """Static particle partition of the reference's MGSP scenes: every model is cut into `world` equal-count slabs along
    `axis`; rank r owns slab r of every model (one model per device in mgsp.cu:34-81; here one slab of each).  A model with
    fewer particles than ranks leaves some slabs empty: those are skipped.  Every part keeps its scene model index in "model"."""
    out = []
    for i, m in enumerate(scene["models"]):
        part = samplers.split_slabs(m["pos"], world, axis)[rank]
        if len(part):
            out.append(dict(material=m["material"], pos=np.ascontiguousarray(part), v0=m["v0"], model=i))
    return dict(domain_bits=scene["domain_bits"], models=out)


def partition_scene_global(scene, rank, world, axis=0):
    """Alternative split: all particles of the scene ordered along `axis`, rank r owns the r-th equal-count slab (each
    rank then holds pieces of the models its slab intersects)."""
    allx = np.concatenate([m["pos"][:, axis] for m in scene["models"]])
    cuts = np.quantile(allx, np.linspace(0, 1, world + 1))
    cuts[0], cuts[-1] = -np.inf, np.inf
    out = []
    for i, m in enumerate(scene["models"]):
        sel = (m["pos"][:, axis] > cuts[rank]) & (m["pos"][:, axis] <= cuts[rank + 1])
        if sel.any():
            out.append(dict(material=m["material"], pos=np.ascontiguousarray(m["pos"][sel]), v0=m["v0"], model=i))
    return dict(domain_bits=scene["domain_bits"], models=out)


def connect(sim, dist=None):
    """Exchange the inbox IPC handles of all ranks and map them (call on every rank before initial_setup)."""
    if sim.mgsp_world <= 1:
        return
    import torch.distributed as td
    dist = dist or td
    handles = [None] * sim.mgsp_world
    dist.all_gather_object(handles, sim.mgsp_ipc_handle())
    sim.mgsp_open_peers(handles)
    dist.barrier()


def common_max_blocks(n_local, dist=None, factor=5.0):
    """Block capacity that EVERY rank must use (the inbox layout is computed from it on both sides of a transfer): sized for the
    largest shard."""
    n = int(n_local)
    if dist is not None and dist.is_initialized():
        import torch
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
        t = torch.tensor([n], dtype=torch.int64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        n = int(t.item())
    return int(max(4000, n / 512 * factor))


def build_rank_sim(scene_part, rank, world, dt, max_blocks, apply_material=None, stream=None, use_graph=True, max_ppc=128, halo_cap=0):
    """One rank's simulator with ITS particle sets registered (MgspBenchmark::init_model(did, positions), mgsp_benchmark.cuh:240-307).
    max_blocks / halo_cap / max_ppc must be the same on every rank (see common_max_blocks).
    apply_material(sim, model_id, material, dx) sets the material parameters (default: claymore_b200.scenes.apply_material)."""
    from . import scenes
    if apply_material is None:
        apply_material = scenes.apply_material
    cfg = Config(domain_bits=scene_part["domain_bits"], max_ppc=max_ppc)
    sim = GmpmSimulator(dt=dt, fps=0, config=cfg, max_blocks=max_blocks, use_graph=use_graph, stream=stream, mgsp_rank=rank, mgsp_world=world, mgsp_halo_cap=halo_cap)
    dx = 1.0 / (1 << scene_part["domain_bits"])
    for m in scene_part["models"]:
        mid = sim.init_model(m["material"], m["pos"], m["v0"])
        try:
            apply_material(sim, mid, m["material"], dx)
        except TypeError:   # test-side helper with the (…, is_oracle) flag
            apply_material(sim, mid, m["material"], dx, False)
    return sim


def partition_scene_grid(scene, rank, world, splits=(2, 2)):
    """2-D static partition: splits[0] equal-count slabs along x, each cut into splits[1] equal-count slabs along y, so that the grid
    blocks around the crossing lines are shared by FOUR ranks (halo sums from three peers)."""
    assert splits[0] * splits[1] == world
    rx, ry = rank // splits[1], rank % splits[1]
    out = []
    for i, m in enumerate(scene["models"]):
        px = samplers.split_slabs(m["pos"], splits[0], 0)[rx]
        py = samplers.split_slabs(px, splits[1], 1)[ry]
        if len(py):
            out.append(dict(material=m["material"], pos=np.ascontiguousarray(py), v0=m["v0"], model=i))
    return dict(domain_bits=scene["domain_bits"], models=out)
