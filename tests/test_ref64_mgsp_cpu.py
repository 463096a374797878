"""The shard comparison (tests/ref64_mgsp.py): its own rejections on synthetic shards built from ref64's output, and the FP32
oracle's halo protocol over N shards against it, which fixes the halo allowance the GPU ranks are held to
(test_gpu_mgsp_ref64.py).
"""
import ctypes as C
import re

import numpy as np
import pytest

import ref64
import ref64_cases as S
import ref64_mgsp as M
from claymore_b200 import mgsp
from claymore_b200._capi import Config
from ref64_checks import BRANCH_MARGIN, DT_ULPS, F_ALLOW, KAPPA, RASTER_KAPPA, STRESS_ALLOW, check_report, rank_models


# ---- splits of a case ------------------------------------------------------------------------------------------------------
def split_case(case, world, kind):
    """Per rank: the case's models cut by ``kind`` ("x": equal-count x-slabs of every model, "2x2": x then y, "global": the scene's
    particles in x-slabs), each part with its scene model index in "model" and the case model's parameters."""
    scene = dict(domain_bits=case["domain_bits"], models=[dict(material=m["material"], pos=m["pos"], v0=m["v0"]) for m in case["models"]])
    out = []
    for r in range(world):
        if kind == "x":
            part = mgsp.partition_scene(scene, r, world)
        elif kind == "2x2":
            part = mgsp.partition_scene_grid(scene, r, world, (2, 2))
        else:
            part = mgsp.partition_scene_global(scene, r, world)
        out.append([dict(case["models"][p["model"]], pos=p["pos"], model=p["model"]) for p in part["models"]])
    return out


# ---- synthetic shards from ref64's own output --------------------------------------------------------------------------------
def synthetic(world=2, seed=3):
    """Random fixed-corotated particles (so that some change particle block), split in x-slabs; every rank's view is the exact
    rasterised grid on its partition.  Returns (cfg, ranks, ref, after): ``after`` follows the protocol exactly: a rank's next
    copy of a key is the reference sum if the key was in its partition, else zero (fresh)."""
    cfg = Config(domain_bits=6)
    dx = 1.0 / 64
    rng = np.random.default_rng(seed)
    pos = rng.uniform(20 * dx, 31 * dx, (3000, 3)).astype(np.float32)
    case = S._case(6, [S.model(S.FIXED_COROTATED, pos, (3.0, -2.0, 1.0), dx)], [0], dt=1e-3)
    parts = split_case(case, world, "x")
    p0 = S.ref_params(case["models"][0])
    fk, fg, _ = ref64.rasterize(cfg, [dict(pos=pos, v0=case["models"][0]["v0"], mass=p0["mass"])])
    full = ref64.Grid(fk, fg)
    ranks = []
    for ps in parts:
        keys = M.partition_keys(cfg, np.concatenate([p["pos"] for p in ps]))
        g, _ = full.gather(keys[:, None, :] * 4 + M._CELLS[None])
        states = [np.concatenate([p["pos"], np.tile(np.eye(3).reshape(1, 9), (len(p["pos"]), 1))], 1) for p in ps]
        ranks.append(dict(keys=keys, grid=g.transpose(0, 2, 1), models=rank_models(ps, states)))
    ref = M.substep(cfg, ranks, case["dt"], case["dt"])
    after = synthetic_after(cfg, ranks, ref)
    return cfg, ranks, ref, after


def synthetic_after(cfg, ranks, ref):
    after = []
    for r, rk in enumerate(ranks):
        states = {gm: mr["state"][~mr["lost"]] for gm, mr in ref["per_rank"][r]}
        keys = M.partition_keys(cfg, np.concatenate(list(states.values()))[:, :3])
        val, _, _ = ref64.ref_at(ref, keys)
        held = np.isin(ref64.key_hash(keys), list(ref["pre_keys"][r]))
        after.append(dict(keys=keys, grid=np.where(held[:, None, None], val, 0.0), states=states))
    return after


@pytest.fixture(scope="module")
def synth():
    return synthetic()


def _compare(cfg, ref, after):
    return M.compare(cfg, ref, after, KAPPA, STRESS_ALLOW, [0.0], margin=BRANCH_MARGIN)


def test_shard_compare_accepts_an_exact_split(synth):
    cfg, ranks, ref, after = synth
    rep = _compare(cfg, ref, after)
    check_report(rep, "exact split")
    assert rep["fresh"] > 0 and rep["max_owners"] == 2, rep   # the synthetic sub-step has fresh copies and shared blocks


def test_shard_compare_rejects_a_missing_owner_in_one_low_weight_cell(synth):
    cfg, ranks, ref, after = synth
    # the cell with the smallest mass among those where both ranks contribute at least a tenth of it
    pk = [ref64.Grid(*p) for p in ref["partials"]]
    cand = []
    for b in np.nonzero((ref["owners"] >= 2).any(1))[0]:
        for c in np.nonzero(ref["owners"][b] >= 2)[0]:
            node = ref["keys"][b] * 4 + M._CELLS[c]
            parts = [p.gather(node[None])[0][0] for p in pk]
            if min(p[0] for p in parts) >= 0.1 * ref["grid"][b, 0, c]:
                cand.append((ref["grid"][b, 0, c], b, c, parts))
    _, b, c, parts = min(cand, key=lambda t: t[0])
    key = ref["keys"][b]
    r = 0
    i = int(np.nonzero(np.all(after[r]["keys"] == key, axis=1))[0][0])
    bad = [dict(a, grid=a["grid"].copy()) for a in after]
    bad[r]["grid"][i, :, c] -= parts[1]                      # rank 0's copy without rank 1's share
    rep = _compare(cfg, ref, bad)
    assert rep["mass"] > 1, rep
    assert rep["worst"]["mass"]["block"] == tuple(int(k) for k in key) and rep["worst"]["mass"]["cell"] == c, rep["worst"]
    with pytest.raises(AssertionError, match=re.escape(f"'block': {tuple(int(k) for k in key)}")):
        check_report(rep, "missing owner")


def test_shard_compare_rejects_a_zero_copy_of_a_block_the_rank_had(synth):
    cfg, ranks, ref, after = synth
    r = 1
    h = ref64.key_hash(after[r]["keys"])
    nz = np.abs(after[r]["grid"]).reshape(len(h), -1).max(1) > 0
    i = int(np.nonzero(nz & np.isin(h, list(ref["pre_keys"][r])))[0][0])
    bad = [dict(a, grid=a["grid"].copy()) for a in after]
    bad[r]["grid"][i] = 0
    key = tuple(int(k) for k in after[r]["keys"][i])
    with pytest.raises(AssertionError, match=rf"rank {r} block {re.escape(str(key))}: all zero, but it was in the rank's partition"):
        _compare(cfg, ref, bad)


def test_shard_compare_rejects_a_fresh_copy_a_particle_reads(synth):
    """Rank 0 without a shared block K in its view before the sub-step (as if K had been fresh there) and with a zero copy of K
    after it: one of its particles reads K at its next G2P, so that zero copy is an error, named by block and particle."""
    cfg, ranks, ref, after = synth
    r = 0
    readers = M._readers(cfg, after[r]["states"])
    h = ref64.key_hash(after[r]["keys"])
    other = set(ref64.key_hash(after[1]["keys"]).tolist())
    i = next(i for i, hh in enumerate(h.tolist()) if hh in readers and hh in other and np.abs(after[1]["grid"][list(ref64.key_hash(after[1]["keys"])).index(hh)]).max() > 0)
    keep = np.ones(len(ranks[r]["keys"]), bool)
    keep[np.nonzero(ref64.key_hash(ranks[r]["keys"]) == h[i])[0]] = False
    pre = [dict(ranks[0], keys=ranks[0]["keys"][keep], grid=ranks[0]["grid"][keep]), ranks[1]]
    ref2 = M.substep(cfg, pre, 1e-3, 1e-3)
    bad = [dict(a, grid=a["grid"].copy()) for a in after]
    bad[r]["grid"][i] = 0
    key = tuple(int(k) for k in after[r]["keys"][i])
    with pytest.raises(AssertionError, match=rf"rank {r} block {re.escape(str(key))}: all zero \(fresh\), but particle \d+ of model 0 at .* reads it"):
        _compare(cfg, ref2, bad)


def test_shard_compare_rejects_a_read_block_missing_from_the_rank(synth):
    """A block one of rank 0's particles reads at its next G2P is absent from rank 0's keys altogether: rejected, named by block and
    particle (the reference could not notice it, since it would gather zeros there as well)."""
    cfg, ranks, ref, after = synth
    r = 0
    readers = M._readers(cfg, after[r]["states"])
    h = ref64.key_hash(after[r]["keys"])
    i = next(i for i, hh in enumerate(h.tolist()) if hh in readers)
    keep = np.arange(len(h)) != i
    bad = [dict(after[0], keys=after[0]["keys"][keep], grid=after[0]["grid"][keep]), after[1]]
    key = tuple(int(k) for k in after[r]["keys"][i])
    with pytest.raises(AssertionError, match=rf"rank {r} block {re.escape(str(key))}: missing from the rank's keys, but particle \d+ of model 0 at .* reads it"):
        _compare(cfg, ref, bad)


def test_shard_dt_rejects_ranks_one_ulp_apart():
    dt = np.float32(7.3e-4)
    M.check_dts([dt, dt, dt], float(dt), DT_ULPS)
    with pytest.raises(AssertionError, match="the ranks' dt differ"):
        M.check_dts([dt, np.nextafter(dt, np.float32(1)), dt], float(dt), DT_ULPS)


# ---- the oracle's halo protocol over N shards ----------------------------------------------------------------------------------
ORACLE_SPLITS = [("fc_cube", 2, "x"), ("fc_cube", 3, "x"), ("fc_cube", 4, "2x2"), ("fluid_cube", 2, "x"), ("multi_model_8", 3, "global"),
                 ("multi_model_8", 3, "x")]


def _halo_exchange(ob, shards, keys, grids):
    """Every shard's blocks that another shard also holds get that shard's copy added (orc_collect_grid_blocks on the sender,
    orc_reduce_grid_blocks on the receiver; every pack is taken before any reduction)."""
    L = ob.lib()
    n = len(shards)
    kh = [set(ref64.key_hash(k).tolist()) for k in keys]
    packs = {}
    for me in range(n):
        for other in range(n):
            if other == me:
                continue
            cfg = shards[me].cfg
            # orc_mark_overlapping_blocks tags against the whole table (exterior blocks included); the halo is the common part of
            # the two neighbour-key sets
            inc = np.ascontiguousarray(keys[other].astype(np.int32).reshape(-1))
            cnt = np.zeros(1, np.int32)
            outk = np.zeros(3 * shards[me].max_blocks, np.int32)
            L.orc_mark_overlapping_blocks(C.byref(cfg), len(keys[other]), other, ob.ptr(inc), shards[me].partition(0), ob.ptr(cnt), ob.ptr(outk))
            tagged = outk[: 3 * int(cnt[0])].reshape(-1, 3)
            common = np.ascontiguousarray(tagged[np.isin(ref64.key_hash(tagged), list(kh[me] & kh[other]))].astype(np.int32))
            assert len(common) == len(kh[me] & kh[other])
            buf = np.zeros(len(common) * 256, np.float32)
            L.orc_collect_grid_blocks(C.byref(cfg), len(common), ob.ptr(common), ob.ptr(grids[other]), shards[other].partition(0), ob.ptr(buf))
            packs[me, other] = (common, buf)
    for (me, other), (common, buf) in sorted(packs.items()):
        L.orc_reduce_grid_blocks(C.byref(shards[me].cfg), len(common), ob.ptr(common), ob.ptr(grids[me]), shards[me].partition(0), ob.ptr(buf))
    return sum(len(c) for c, _ in packs.values())


def oracle_shards_check(ob, name, world, kind):
    """Set-up rasterisation and the first sub-step of the case's shards on the oracle, halo sums exchanged after each, against
    ref64 through the shard comparison.  Returns the reports (set-up, sub-step)."""
    case = S.CASES[name]
    parts = split_case(case, world, kind)
    shards = [S.build_oracle(ob, dict(case, models=ps)) for ps in parts]
    cfg = shards[0].cfg
    counts = [s.block_counts() for s in shards]
    keys = [s.partition_arrays(0)["active_keys"][: 3 * nbc].reshape(-1, 3).astype(np.int64) for s, (_, nbc, _) in zip(shards, counts)]
    g0 = [s.grid_array(0) for s in shards]
    g1 = [s.grid_array(1) for s in shards]
    assert _halo_exchange(ob, shards, keys, g0) > 0
    views = [g[: len(k) * 256].reshape(-1, 4, 64).astype(np.float64) for g, k in zip(g0, keys)]
    # set-up
    ref = M.rasterize(cfg, [[dict(pos=p["pos"], v0=p["v0"], mass=S.ref_params(p)["mass"]) for p in ps] for ps in parts])
    setup_after = [dict(keys=k, grid=v) for k, v in zip(keys, views)]
    rep_setup = M.compare(cfg, ref, setup_after, RASTER_KAPPA, 0.0, [])
    rep_setup["halo_worst"] = halo_worst(ref, setup_after, RASTER_KAPPA, 0.0)
    # the first sub-step: every shard's grid update, the max over the shards, g2p2g of every model, the halo sums
    dt = shards[0].dt
    ranks = [dict(keys=k, grid=v, models=rank_models(ps, [s.particle_state(i) for i in range(len(ps))])) for k, v, ps, s in zip(keys, views, parts, shards)]
    r = M.substep(cfg, ranks, dt, case["dt"], n_models=len(case["models"]))
    L = ob.lib()
    mx = 0.0
    for s, (_, nbc, _) in zip(shards, counts):
        mv = np.zeros(1, np.float32)
        L.orc_update_grid_velocity_query_max(C.byref(cfg), nbc, ob.ptr(s.grid_array(0)), s.partition_arrays(0)["struct"], dt, ob.ptr(mv))
        mx = max(mx, float(mv[0]))
    new_dt = float(np.float32(ref64.compute_dt(cfg, mx, case["dt"])))
    after = []
    for s, (pbc, nbc, ebc), k, ps in zip(shards, counts, keys, parts):
        s.grid_array(1)[: nbc * 256] = 0
        states = {}
        for i, p in enumerate(ps):
            cur, nxt = s.buffer_arrays(i, 0), s.buffer_arrays(i, 1)
            nxt["cell_particle_counts"][: ebc * 64] = 0
            L.orc_g2p2g(C.byref(cfg), dt, new_dt, pbc, cur["struct"], nxt["struct"], s.partition_arrays(1)["struct"], s.partition_arrays(0)["struct"],
                        ob.ptr(s.grid_array(0)), ob.ptr(s.grid_array(1)))
            states[p["model"]] = S.states_from_bins(nxt["bins"], nxt["bin_offsets"], nxt["particle_bucket_sizes"], pbc, p["material"])
        after.append(dict(keys=k, states=states))
    _halo_exchange(ob, shards, keys, g1)
    for a, g in zip(after, g1):
        a["grid"] = g[: len(a["keys"]) * 256].reshape(-1, 4, 64).astype(np.float64)
    rep = M.compare(cfg, r, after, KAPPA, STRESS_ALLOW, [F_ALLOW[m["material"]] for m in case["models"]], margin=BRANCH_MARGIN)
    rep["halo_worst"] = halo_worst(r, after, KAPPA, STRESS_ALLOW)
    M.check_dts([new_dt], r["new_dt"], DT_ULPS)
    for s in shards:
        s.close()
    return rep_setup, rep


def halo_worst(ref, after, kappa, stress_allow):
    """The worst |copy - ref| / bound over the cells with two or more owners, with the plain kappa bound (no halo allowance)."""
    w = 0.0
    for a in after:
        val, mag, st, own = M._ref_at(ref, a["keys"])
        err = np.abs(np.asarray(a["grid"], np.float64) - val)
        for c, q, sa in ((slice(0, 1), "mass", 0.0), (slice(1, 4), "momentum", stress_allow)):
            bound = kappa[q] * ref64.EPS32 * mag[:, c] + sa * st[:, c]
            m = (own[:, None, :] >= 2) & (bound > 0)
            if m.any():
                w = max(w, float((err[:, c][m] / bound[m]).max()))
    return w


@pytest.mark.parametrize("name,world,kind", ORACLE_SPLITS, ids=[f"{n}-{w}{k}" for n, w, k in ORACLE_SPLITS])
def test_oracle_shards_match_ref64(oracle, name, world, kind):
    rep_setup, rep = oracle_shards_check(oracle, name, world, kind)
    check_report(rep_setup, f"{name} {world} {kind} set-up")
    check_report(rep, f"{name} {world} {kind} sub-step 0")
    assert rep["max_owners"] >= (4 if kind == "2x2" else 2), rep
    # cells with several owners, against the single-domain bound with no halo allowance: compared, and within it
    for r, q in ((rep_setup, "set-up"), (rep, "sub-step")):
        assert 0 < r["halo_worst"] <= 1.0, (q, r["halo_worst"])
    print(f"{name} {world} {kind}: set-up mass {rep_setup['mass']:.3g} momentum {rep_setup['momentum']:.3g}; sub-step mass {rep['mass']:.3g} "
          f"momentum {rep['momentum']:.3g} pos {rep['pos']:.3g} F {rep['F']:.3g}; max owners {rep['max_owners']}; cells with 2+ owners: "
          f"{rep_setup['halo_worst']:.3g} (set-up) {rep['halo_worst']:.3g} (sub-step) of the kappa bound")
