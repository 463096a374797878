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

     "boundaries": [{"shape": "plane"|"box"|"sphere"|"cylinder", + the "collider" keys offset, span, normal, type, friction,
                     velocity, omega, scale, dsdt}, ...]

Analytic collision objects (claymore_b200.objects, DESIGN.md section 2.9), resolved after the collider in list order, at most
CB200_MAX_COLLISION_OBJECTS.  Box, sphere and plane are placed as the collider's are; a "cylinder" fills [offset, offset + span]
with its axis along y and radius min(span_x, span_z) / 2.  {"shape": "levelset", "file": "<name>.sdf"} is an SDFGen level set fitted
into [offset, offset + span] as a model's is (DESIGN.md section 2.11), but it may extend past the domain; each file is read once and
its lattice registered once per simulator.  Unknown keys or shapes, too many entries, an unreadable file or a bad value raise
ValueError before any device work; "collider" and "boundaries" may both be present.

A "boundaries" entry may move on a keyframed track (claymore_b200.objects.track, DESIGN.md section 2.14):

     "track": {"keys": [{"t": 0.0, "position": [3], "rotation": [3]}, ...], "interp": "linear"|"smooth", "periodic": false}

The pivot of a tracked entry is the centre of its [offset, offset + span] box (for a plane: offset); the shape is placed as it is
without a track and turned and moved about that pivot.  "position" is where the pivot is at time "t" (default: where it is placed,
the centre), "rotation" a rotation vector in radians (default [0, 0, 0]), applied in world space after the entry's rest orientation;
a "scale" scales the shape about the pivot.
A tracked entry has no "velocity", "omega" or "dsdt"; a bad track raises ValueError before any device work.

A "file": "<name>.obj" model, boundary or sink is a Wavefront OBJ triangle mesh turned into a level set on the device
(claymore_b200.mesh, SDFGen's make_level_set3 bit for bit, DESIGN.md section 2.12) with the optional keys "h" (node spacing in mesh
units; default: the mesh's longest extent x dx / the longest span, about one simulation cell per level-set cell), "padding" (1) and
"exact_band" (1); from there it is an `.sdf` level set in every respect.  Each distinct (file, h, padding, exact_band) is built
once, after every file has been read and every entry validated, and registered once.

The reference only loads `.sdf` level sets (gmpm.cu:152-159).  Here "file": "<name>.sdf" is sampled on the device by
GmpmSimulator.init_model_sdf with the optional keys "sampler" ("random", the default, or "lattice"), "ppc" (particles per
simulation cell, default 8: the reference's MODEL_PPC, settings.h:51) and "seed" (default 0); the level set is fitted into
[offset, offset + span] with one scale for all axes, and a node box outside the domain rejects the scene before any device work
(claymore_b200.sdf).  A model may also name a synthetic generator: "file": "box" (span in cells of the lattice sampler) or
"sphere" (span = diameter), or a raw float32 xyz `.bin` cloud as used by mgsp.cu:11-17.

A model may be a source: "emit": {"start": 2, "every": 1, "until": <frames>, "fill": "all"|"empty"} (defaults as shown; "until"
defaults to the scene's frame count).  At the start of frames start, start + every, ... <= until, before the frame's sub-steps, the
model's own shape (its file / offset / span, or its `.sdf` level set with its sampler and ppc; random mode with seed seed + frame) is
sampled again and added with the model's "velocity" (GmpmSimulator.add_particles).  "fill": "empty" adds only particles whose cell
holds no particle, so a repeating source refills only the cells its material has left.  Frame 1 starts from the model's initial
particles; a resumed run emits exactly the frames an uninterrupted run emits after the checkpoint's frame.  Bad "emit" keys or
values, or "emit" in MGSP mode, raise ValueError before any device work.

     "sinks": [{"shape", "offset", "span", "normal", "velocity", "omega", "scale", "dsdt", "models": [...], "outside": false,
                "start": 1, "every": 1, "until": <frames>}, ...]

Outlets (GmpmSimulator.remove_particles, DESIGN.md section 2.10).  A sink's region is placed as a "boundaries" entry of its shape is
placed, at the simulated time; "models" (scene model indices) defaults to all of them, and "outside": true removes what lies outside
the region instead of inside it.  At the start of frames start, start + every, ... <= until ("until" defaults to the scene's frame
count), before the sources emit, the sinks due at that frame with the same "models" and "outside" are removed in one call (at most
CB200_MAX_COLLISION_OBJECTS sinks in one such group).  A resumed run applies exactly the frames after the checkpoint's frame.  Bad
keys or values, too many sinks in one group, or "sinks" in MGSP mode raise ValueError before any device work.
"""
import csv
import json
import os

import numpy as np

from . import levelset, mesh, samplers, sdf
from ._capi import Config, FIXED_COROTATED, J_FLUID, NACC, SAND
from .simulator import GmpmSimulator

CONSTITUTIVE = {"jfluid": J_FLUID, "fixed_corotated": FIXED_COROTATED, "sand": SAND, "nacc": NACC}
PARTICLE_TYPES = ("particles", "particle")   # the reference's scene.json says "particle"; gmpm.cu:96-165 does not read the key


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
    raise ValueError(f"unsupported model file {kind!r} (known: box, sphere, *.sdf, *.obj, *.bin, *.npy)")


def _model_path(model, base_dir):
    kind = model.get("file", "box")
    return kind if os.path.isabs(kind) else os.path.join(base_dir, kind)


MESH_KEYS = ("h", "padding", "exact_band")   # with a "file": "*.obj" model, boundary or sink


def _mesh_level_set(e, path, what, span, dx, cache):
    """The level set of the `.obj` entry `e`, one per (path, h, padding, exact_band) in `cache`: read and checked on the host here, its
    phi left None until _build_level_sets (ValueError naming `what`).  h defaults to the mesh's longest extent x dx / the longest
    span, so that one level-set cell is about one simulation cell."""
    try:
        if ("obj", path) not in cache:
            cache[("obj", path)] = mesh.read_obj(path)
        m = cache[("obj", path)]
        lo, hi = m.bounds if len(m.vertices) else (np.zeros(3), np.zeros(3))
        h = e.get("h", float(np.max(hi - lo)) * dx / max(sdf._vec3(span)))
        padding, band = e.get("padding", 1), e.get("exact_band", 1)
        for k, v in (("h", h), ("padding", padding), ("exact_band", band)):
            if isinstance(v, bool) or not isinstance(v, (int, float)) or (k != "h" and not isinstance(v, int)):
                raise ValueError(f"\"{k}\" must be a {'number' if k == 'h' else 'integer'}, not {v!r}")
        key = (path, float(np.float32(h)), padding, band)
        if key not in cache:
            ls = sdf.LevelSet(mesh.header(m, h, padding, band), None)
            ls.source = (m, h, padding, band)
            cache[key] = ls
        return cache[key]
    except (OSError, ValueError) as e:
        raise ValueError(f"{what}: {os.path.basename(path)}: {e}") from None


def _build_level_sets(cache):
    """Builds, on the current device, every mesh level set of `cache` that has no phi yet (each distinct one once)."""
    for ls in cache.values():
        if isinstance(ls, sdf.LevelSet) and ls.phi is None:
            built = mesh.levelset(*ls.source)
            ls.header, ls.phi = built.header, built.phi


def _level_sets(models, base_dir, dx=None, cache=None):
    """Reads every `.sdf` model's level set and every `.obj` model's mesh and checks its node box: {model index: LevelSet}, before any
    device work.  A mesh's level set is built later by _build_level_sets(cache)."""
    out = {}
    dx = Config().dx if dx is None else dx
    cache = {} if cache is None else cache
    for i, model in enumerate(models):
        f = str(model.get("file", "box"))
        if f.endswith(".obj"):
            ls = _mesh_level_set(model, _model_path(model, base_dir), f"model {i}", model.get("span", [1, 1, 1]), dx, cache)
        if f.endswith(".sdf") or f.endswith(".obj"):
            if f.endswith(".sdf"):
                ls = sdf.read(_model_path(model, base_dir))
            sdf.check_box(ls, model.get("offset", [0, 0, 0]), model.get("span", [1, 1, 1]), what=f"model {i} ({model['file']})")
            sdf.sampling(model.get("offset", [0, 0, 0]), model.get("span", [1, 1, 1]), model.get("ppc", 8), model.get("sampler", "random"),
                         model.get("seed", 0))
            out[i] = ls
    return out


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


BOUNDARY_KEYS = ("shape", "offset", "span", "normal", "type", "friction", "velocity", "omega", "scale", "dsdt", "track")
TRACK_KEYS = ("keys", "interp", "periodic")
TRACK_KEY_KEYS = ("t", "position", "rotation")


def _track(tr, pivot):
    """objects.track of a "track" entry whose keys' positions default to pivot and whose rotations are rotation vectors (ValueError on a
    bad entry)."""
    from . import objects
    if not isinstance(tr, dict):
        raise ValueError(f"\"track\" must be an object with keys {', '.join(TRACK_KEYS)}")
    unknown = sorted(set(tr) - set(TRACK_KEYS))
    if unknown:
        raise ValueError(f"track: unknown keys {unknown} (known: {', '.join(TRACK_KEYS)})")
    keys = tr.get("keys")
    if not isinstance(keys, list) or not keys:
        raise ValueError("track: \"keys\" must be a non-empty list")
    out = []
    for k, key in enumerate(keys):
        if not isinstance(key, dict) or "t" not in key:
            raise ValueError(f"track key {k} must be an object with \"t\" and optional \"position\", \"rotation\"")
        unknown = sorted(set(key) - set(TRACK_KEY_KEYS))
        if unknown:
            raise ValueError(f"track key {k}: unknown keys {unknown} (known: {', '.join(TRACK_KEY_KEYS)})")
        r = np.asarray(key.get("rotation", [0.0, 0.0, 0.0]), np.float64).reshape(3)
        th = float(np.linalg.norm(r))
        q = [1.0, 0.0, 0.0, 0.0] if th == 0.0 else [np.cos(th / 2)] + list(np.sin(th / 2) * r / th)
        out.append((float(key["t"]), np.asarray(key.get("position", pivot), np.float64).reshape(3), q))
    if not isinstance(tr.get("periodic", False), bool):
        raise ValueError("track: \"periodic\" must be true or false")
    return objects.track(out, tr.get("interp", "linear"), tr.get("periodic", False))
LEVELSET_KEYS = ("file",) + MESH_KEYS   # with "shape": "levelset"


def _obstacle_level_set(b, what, base_dir, cache, span=(1, 1, 1), dx=None):
    """The sdf.LevelSet of a "levelset" entry, read once per path (an .obj mesh: once per path, h, padding and band) into `cache`
    (ValueError naming `what` on a bad file)."""
    f = b.get("file")
    if not isinstance(f, str) or not (f.endswith(".sdf") or f.endswith(".obj")):
        raise ValueError(f"{what} (levelset): \"file\" must name an .sdf level set or an .obj mesh, not {f!r}")
    path = f if os.path.isabs(f) else os.path.join(base_dir if base_dir is not None else os.getcwd(), f)
    if f.endswith(".obj"):
        return _mesh_level_set(b, path, f"{what} (levelset)", span, Config().dx if dx is None else dx, cache)
    if any(k in b for k in MESH_KEYS):
        raise ValueError(f"{what} (levelset): {', '.join(k for k in MESH_KEYS if k in b)} only apply to an .obj mesh")
    if path not in cache:
        try:
            cache[path] = sdf.read(path)
        except (OSError, ValueError) as e:
            raise ValueError(f"{what} (levelset): {f}: {e}") from None
    return cache[path]


def _object(b, what, keys, base_dir=None, cache=None, dx=None):
    """The collision object of one "boundaries" or "sinks" entry `b` (ValueError naming `what` on a bad entry or a key not in `keys`).
    A "levelset" entry's file is read through `cache` ({path: LevelSet}), so that one file is one level set."""
    from . import objects
    if not isinstance(b, dict):
        raise ValueError(f"{what} must be an object with keys {', '.join(keys)}")
    shape = b.get("shape")
    if shape == "levelset":
        keys = tuple(keys) + LEVELSET_KEYS
    unknown = sorted(set(b) - set(keys))
    if unknown:
        raise ValueError(f"{what}: unknown keys {unknown} (known: {', '.join(keys)})")
    if shape not in objects.SHAPES and shape != "levelset":
        raise ValueError(f"{what}: unknown shape {shape!r} (known: {', '.join(objects.SHAPES)}, levelset)")
    try:
        offset = np.asarray(b.get("offset", [0, 0, 0]), dtype=np.float64).reshape(3)
        span = np.asarray(b.get("span", [1, 1, 1]), dtype=np.float64).reshape(3)
        motion = dict(type=b.get("type", "sticky"), friction=float(b.get("friction", 0.3)), trans_vel=b.get("velocity", [0, 0, 0]),
                      omega=b.get("omega", [0, 0, 0]), scale=float(b.get("scale", 1.0)), dsdt=float(b.get("dsdt", 0.0)))
        if "track" in b:  # placed about its pivot: x = R(t)^T (p - c(t)) scale + pivot, the rest pose at c = pivot is the untracked one
            pivot = offset if shape == "plane" else offset + span / 2
            motion.update(trans=pivot, track=_track(b["track"], pivot))
        if shape == "levelset":
            ls = _obstacle_level_set(b, what, base_dir, {} if cache is None else cache, span, dx)
            return objects.levelset(ls, offset, span, **motion)
        if shape == "box":
            return objects.box(offset, offset + span, **motion)
        if shape == "sphere":
            return objects.sphere(offset + span / 2, float(span.min()) / 2, **motion)
        if shape == "plane":
            return objects.plane(offset, b.get("normal", [0, 1, 0]), **motion)
        return objects.cylinder(offset + span / 2, float(min(span[0], span[2])) / 2, float(span[1]) / 2, **motion)
    except (TypeError, ValueError) as e:
        raise ValueError(f"{what} ({shape}): {e}") from None


def boundaries(doc, base_dir=None, cache=None, dx=None):
    """The scene's "boundaries" as validated collision objects (ValueError on a bad entry), before any device work.  Level-set files
    are relative to base_dir (default: the working directory) and read through `cache` ({path: LevelSet}); dx (default: Config's)
    sets an .obj mesh's default h."""
    from . import objects
    bs = doc.get("boundaries", [])
    if not isinstance(bs, list):
        raise ValueError("\"boundaries\" must be a list of objects")
    if len(bs) > objects.MAX_COLLISION_OBJECTS:
        raise ValueError(f"at most {objects.MAX_COLLISION_OBJECTS} \"boundaries\", not {len(bs)}")
    return [_object(b, f"boundary {i}", BOUNDARY_KEYS, base_dir, cache, dx) for i, b in enumerate(bs)]


SINK_KEYS = ("shape", "offset", "span", "normal", "velocity", "omega", "scale", "dsdt", "models", "outside", "start", "every", "until")


def sinks(doc, base_dir=None, cache=None, dx=None):
    """The scene's validated "sinks": [{"object", "models" (sorted tuple of scene model indices), "outside", "frames" (list)}], in
    document order (ValueError on a bad entry, or on more than CB200_MAX_COLLISION_OBJECTS sinks due in one group), before any
    device work.  base_dir and cache: as for boundaries."""
    from . import objects
    frames = doc.get("simulation", {}).get("frames", GmpmSimulator.DEFAULT_FRAMES)
    n_models = len([m for m in doc.get("models", []) if m.get("type", "particles") in PARTICLE_TYPES])
    ss = doc.get("sinks", [])
    if not isinstance(ss, list):
        raise ValueError("\"sinks\" must be a list of objects")
    out = []
    for i, e in enumerate(ss):
        what = f"sink {i}"
        o = _object(e, what, SINK_KEYS, base_dir, cache, dx)
        models = e.get("models", list(range(n_models)))
        if not isinstance(models, list) or not models:
            raise ValueError(f"{what}: \"models\" must be a non-empty list of model indices, not {models!r}")
        for m in models:
            if isinstance(m, bool) or not isinstance(m, int) or not 0 <= m < n_models:
                raise ValueError(f"{what}: unknown model {m!r} (the scene has {n_models})")
        outside = e.get("outside", False)
        if not isinstance(outside, bool):
            raise ValueError(f"{what}: \"outside\" must be true or false, not {outside!r}")
        spec = {k: e.get(k, d) for k, d in (("start", 1), ("every", 1), ("until", None))}
        if spec["until"] is None:   # the last frame; a scene shorter than `start` then never removes
            spec["until"] = max(frames, spec["start"]) if isinstance(spec["start"], int) else frames
        for k, v in spec.items():
            if isinstance(v, bool) or not isinstance(v, int):
                raise ValueError(f"{what}: \"{k}\" must be an integer, not {v!r}")
        if spec["start"] < 1:
            raise ValueError(f"{what}: \"start\" must be at least 1, not {spec['start']}")
        if spec["every"] < 1:
            raise ValueError(f"{what}: \"every\" must be at least 1, not {spec['every']}")
        if spec["until"] < spec["start"]:
            raise ValueError(f"{what}: \"until\" ({spec['until']}) must not precede \"start\" ({spec['start']})")
        out.append({"object": o, "models": tuple(sorted(set(models))), "outside": outside,
                    "frames": list(range(spec["start"], min(spec["until"], frames) + 1, spec["every"]))})
    for f, groups in _sink_groups(out).items():
        for (models, outside), idx in groups.items():
            if len(idx) > objects.MAX_COLLISION_OBJECTS:
                raise ValueError(f"frame {f}: {len(idx)} sinks of models {list(models)} (outside={outside}) are due together; at most "
                                 f"{objects.MAX_COLLISION_OBJECTS}")
    return out


def _sink_groups(specs, after=0):
    """{frame: {(models, outside): [sink indices]}} over the frames > after, groups and indices in document order."""
    out = {}
    for i, sp in enumerate(specs):
        for f in sp["frames"]:
            if f > after:
                out.setdefault(f, {}).setdefault((sp["models"], sp["outside"]), []).append(i)
    return dict(sorted(out.items()))


def sink_schedule(doc, after=0, base_dir=None, cache=None, dx=None):
    """{frame: [(models, outside, [sink indices]), ...]}: the removal calls of every frame > `after` (a resumed run's checkpoint
    frame), one per group of sinks due together with the same models and outside, in document order.  Validates "sinks"."""
    return {f: [(m, o, idx) for (m, o), idx in g.items()] for f, g in _sink_groups(sinks(doc, base_dir, cache, dx), after).items()}


def _sink_hook(doc, after=0, base_dir=None, cache=None, dx=None):
    """main_loop's per-frame hook that applies the scene's sinks (None without any), built before any device work."""
    specs = sinks(doc, base_dir, cache, dx)
    todo = sink_schedule(doc, after, base_dir, cache, dx)
    if not todo:
        return None

    def remove(s, f):
        for models, outside, idx in todo.get(f, ()):
            s.remove_particles([specs[i]["object"] for i in idx], models=models, outside=outside)
    return remove


EMIT_KEYS = ("start", "every", "until", "fill")
EMIT_FILLS = ("all", "empty")


def _emit_spec(model, i, frames):
    """The validated "emit" entry of scene model i (None without one): {"start", "every", "until", "fill"}."""
    e = model.get("emit")
    if e is None:
        return None
    if not isinstance(e, dict):
        raise ValueError(f"model {i}: \"emit\" must be an object with keys {', '.join(EMIT_KEYS)}")
    unknown = sorted(set(e) - set(EMIT_KEYS))
    if unknown:
        raise ValueError(f"model {i}: unknown \"emit\" keys {unknown} (known: {', '.join(EMIT_KEYS)})")
    spec = {"start": e.get("start", 2), "every": e.get("every", 1), "until": e.get("until"), "fill": e.get("fill", "all")}
    if spec["until"] is None:   # the last frame; a scene shorter than `start` then has no emission
        spec["until"] = max(frames, spec["start"]) if isinstance(spec["start"], int) else frames
    for k in ("start", "every", "until"):
        if isinstance(spec[k], bool) or not isinstance(spec[k], int):
            raise ValueError(f"model {i}: \"emit\".{k} must be an integer, not {spec[k]!r}")
    if spec["every"] < 1:
        raise ValueError(f"model {i}: \"emit\".every must be at least 1, not {spec['every']}")
    if spec["start"] < 2:
        raise ValueError(f"model {i}: \"emit\".start must be at least 2 (frame 1 starts from the initial particles), not {spec['start']}")
    if spec["until"] < spec["start"]:
        raise ValueError(f"model {i}: \"emit\".until ({spec['until']}) must not precede start ({spec['start']})")
    if spec["fill"] not in EMIT_FILLS:
        raise ValueError(f"model {i}: unknown \"emit\".fill {spec['fill']!r} (known: {', '.join(EMIT_FILLS)})")
    return spec


def emit_schedule(doc, after=0):
    """{scene model index: [(frame, seed), ...]}: the emissions of every source model at frames > `after` (a resumed run's checkpoint
    frame), with the seed its random-mode sampling uses.  Validates every "emit" entry (ValueError)."""
    frames = doc.get("simulation", {}).get("frames", GmpmSimulator.DEFAULT_FRAMES)
    models = [m for m in doc.get("models", []) if m.get("type", "particles") in PARTICLE_TYPES]
    out = {}
    for i, model in enumerate(models):
        spec = _emit_spec(model, i, frames)
        if spec is not None:
            seed = model.get("seed", 0)
            out[i] = [(f, seed + f) for f in range(spec["start"], min(spec["until"], frames) + 1, spec["every"]) if f > after]
    return out


def _emitters(doc, cfg, base, level_sets):
    """main_loop's per-frame emitters of the scene's source models (every source file is read here, before any device work)."""
    frames = doc.get("simulation", {}).get("frames", GmpmSimulator.DEFAULT_FRAMES)
    models = [m for m in doc.get("models", []) if m.get("type", "particles") in PARTICLE_TYPES]
    out = []
    for i, frames_seeds in emit_schedule(doc).items():
        model = models[i]
        todo = dict(frames_seeds)
        v0, fill = model.get("velocity", [0, 0, 0]), _emit_spec(model, i, frames)["fill"]
        offset, span = model.get("offset", [0, 0, 0]), model.get("span", [1, 1, 1])
        if i in level_sets:
            ls, ppc, mode = level_sets[i], model.get("ppc", 8), model.get("sampler", "random")

            def emit(s, f, i=i, ls=ls, ppc=ppc, mode=mode, todo=todo, v0=v0, fill=fill, offset=offset, span=span):
                if f in todo:
                    s.add_particles_sdf(i, ls, offset, span, v0, ppc=ppc, mode=mode, seed=todo[f], fill=fill)
        else:
            pos = _positions(model, cfg, base)

            def emit(s, f, i=i, pos=pos, todo=todo, v0=v0, fill=fill):
                if f in todo:
                    s.add_particles(i, pos, v0, fill=fill)
        out.append(emit)
    return out


def _check_resume(doc, cfg, resume):
    """The checkpoint `resume` must belong to this document: same config, default dt, fps and constitutive models."""
    from . import checkpoint
    inf = checkpoint.info(resume)
    s = doc.get("simulation", {})
    f32 = lambda v: float(np.float32(v))
    want = dict(domain_bits=cfg.domain_bits, max_ppc=cfg.max_ppc, boundary=cfg.boundary, gravity=f32(cfg.gravity), cfl=f32(cfg.cfl))
    if inf["cfg"] != want:
        raise ValueError(f"checkpoint {resume}: config {inf['cfg']} differs from the scene's {want}")
    if inf["dt_default"] != f32(s.get("default_dt", GmpmSimulator.DEFAULT_DT)) or inf["fps"] != s.get("fps", GmpmSimulator.DEFAULT_FPS):
        raise ValueError(f"checkpoint {resume}: default_dt / fps {inf['dt_default']} / {inf['fps']} differ from the scene's simulation section")
    mats = [CONSTITUTIVE.get(m.get("constitutive")) for m in doc.get("models", []) if m.get("type", "particles") in PARTICLE_TYPES]
    if [m["material"] for m in inf["models"]] != mats:
        raise ValueError(f"checkpoint {resume}: its models are not the scene's")
    return inf


FORCE_COLUMNS = ("frame", "time", "body", "shape", "Fx", "Fy", "Fz", "Tx", "Ty", "Tz")


def force_bodies(doc):
    """The shape of each body of the impulse report: the "collider" (body 0, "none" without one), then the "boundaries" entries in
    document order."""
    return ["collider" if "collider" in doc else "none"] + [b.get("shape", "") for b in doc.get("boundaries", [])]


def force_recorder(sim, path, append=False):
    """(on_frame, file): main_loop's per-frame hook that writes one CSV row per body of sim.force_bodies to `path` (FORCE_COLUMNS): the
    frame, the simulated time at its end and the mean force and torque over the frame, the impulses read and reset once per frame.
    append: continue the file of an interrupted run (a resumed run's frames follow its checkpoint's); else it is truncated."""
    f = open(path, "a" if append else "w", newline="")
    w = csv.writer(f)
    if f.tell() == 0:
        w.writerow(FORCE_COLUMNS)
    shapes = sim.force_bodies

    def on_frame(s, frame):
        elapsed, imp = s.collision_forces()
        t = s.sim_time()
        mean = imp / elapsed if elapsed > 0 else np.zeros_like(imp)
        for k, row in enumerate(mean):
            w.writerow([frame, "%.17g" % t, k, shapes[k]] + ["%.17g" % x for x in row])
        f.flush()
    return on_frame, f


def parse_scene(path_or_dict, config=None, max_blocks=10000, resume=None, forces=False, **sim_kwargs):
    """parse_scene (gmpm.cu:60-165): returns an initialised GmpmSimulator with every model registered.
    resume: path of a checkpoint of this scene.  It is checked against the document before any simulator exists; the scene's
    collider and boundaries are set and the checkpoint restored in place of the models (max_blocks defaults to the saved capacity).  MGSP runs
    resume rank by rank instead: GmpmSimulator.from_checkpoint, wire the peers, restore.
    forces: turn on the boundary impulse report (GmpmSimulator.report_forces); sim.force_bodies names its bodies (force_bodies).  Not
    in MGSP mode (ValueError)."""
    if isinstance(path_or_dict, dict):
        doc, base = path_or_dict, os.getcwd()
    else:
        with open(path_or_dict) as f:
            doc = json.load(f)
        base = os.path.dirname(os.path.abspath(path_or_dict))
    cfg = config if config is not None else Config()
    s = doc.get("simulation", {})
    if emit_schedule(doc) and sim_kwargs.get("mgsp_world", 1) > 1:
        raise ValueError("\"emit\" is not supported in MGSP mode")
    if doc.get("sinks") and sim_kwargs.get("mgsp_world", 1) > 1:
        raise ValueError("\"sinks\" are not supported in MGSP mode")
    if forces and sim_kwargs.get("mgsp_world", 1) > 1:
        raise ValueError("the force report is not supported in MGSP mode by the scene runner")
    models = [m for m in doc.get("models", []) if m.get("type", "particles") in PARTICLE_TYPES]
    # {path or (path, h, padding, band): LevelSet} of the "levelset" boundaries and sinks and the .obj models: one build and one
    # registration per distinct level set
    obstacles = {}
    objs = boundaries(doc, base, obstacles, cfg.dx)
    if resume is not None:
        inf = _check_resume(doc, cfg, resume)
        emitters = _emitters(doc, cfg, base, _level_sets(models, base, cfg.dx, obstacles))
        sink = _sink_hook(doc, inf["frames"], base, obstacles, cfg.dx)
        _build_level_sets(obstacles)   # deterministic: the same phi as the run that wrote the checkpoint
        sim = GmpmSimulator(gpu=s.get("gpuid", 0), dt=s.get("default_dt", GmpmSimulator.DEFAULT_DT), fps=s.get("fps", GmpmSimulator.DEFAULT_FPS),
                            frames=s.get("frames", GmpmSimulator.DEFAULT_FRAMES), config=cfg, max_blocks=max(max_blocks, inf["max_blocks"]), **sim_kwargs)
        if "collider" in doc:
            _collider(sim, doc["collider"], cfg, base)
        if objs:
            sim.set_collision_objects(objs)
        sim.restore(resume)
        sim.emitters = ([sink] if sink else []) + emitters
        _report_forces(sim, doc, forces)
        return sim
    for model in models:
        if model.get("constitutive") not in CONSTITUTIVE:
            raise ValueError(f"unknown constitutive model {model.get('constitutive')!r}")
    level_sets = _level_sets(models, base, cfg.dx, obstacles)
    sink = _sink_hook(doc, 0, base, obstacles, cfg.dx)
    emitters = _emitters(doc, cfg, base, level_sets)
    _build_level_sets(obstacles)
    sim = GmpmSimulator(gpu=s.get("gpuid", 0), dt=s.get("default_dt", GmpmSimulator.DEFAULT_DT), fps=s.get("fps", GmpmSimulator.DEFAULT_FPS),
                        frames=s.get("frames", GmpmSimulator.DEFAULT_FRAMES), config=cfg, max_blocks=max_blocks, **sim_kwargs)
    for i, model in enumerate(models):
        c = model["constitutive"]
        v0 = model.get("velocity", [0, 0, 0])
        if i in level_sets:
            mid = sim.init_model_sdf(CONSTITUTIVE[c], level_sets[i], model.get("offset", [0, 0, 0]), model.get("span", [1, 1, 1]), v0,
                                     ppc=model.get("ppc", 8), mode=model.get("sampler", "random"), seed=model.get("seed", 0))
        else:
            mid = sim.init_model(CONSTITUTIVE[c], _positions(model, cfg, base), v0)
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
    if objs:
        sim.set_collision_objects(objs)
    sim.emitters = ([sink] if sink else []) + emitters
    _report_forces(sim, doc, forces)
    return sim


def _report_forces(sim, doc, forces):
    sim.force_bodies = force_bodies(doc)
    if forces:
        sim.report_forces(True)
