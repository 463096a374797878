"""The scene runner, the reference's `gmpm -f scene.json` (Projects/GMPM/gmpm.cu):

    python -m claymore_b200 -f scene.json [--out DIR] [--attributes v,J] [--resume CKPT] [--forces]

parse_scene, then main_loop: every finished frame is written to DIR (default: the working directory) as
model_id[i]_frame[f].bgeo, with the per-particle attributes listed (v: velocity, J: volume ratio).  --resume continues a
checkpoint of the same scene and writes only its remaining frames.  --forces also writes DIR/forces.csv: per finished frame and
body (0: the "collider", then the "boundaries" in document order) the mean force and torque the material exerted on it over the
frame (scene.force_recorder); a resumed run appends its frames' rows, a fresh run truncates the file.

    python -m claymore_b200 mesh2sdf in.obj out.sdf --h H [--padding P] [--exact-band B]

builds the level set of a triangle mesh on the GPU (claymore_b200.mesh: SDFGen's make_level_set3, bit for bit) and writes it as
SDFGen text with 9 significant digits, in place of running SDFGen by hand.
"""
import argparse
import os
import sys

from .scene import force_recorder, parse_scene


def mesh2sdf(argv):
    from . import mesh, sdf
    ap = argparse.ArgumentParser(prog="python -m claymore_b200 mesh2sdf", description="Write the level set of an .obj mesh as an .sdf file.")
    ap.add_argument("obj", help="Wavefront OBJ triangle mesh")
    ap.add_argument("sdf", help="output SDFGen level set")
    ap.add_argument("--h", type=float, required=True, help="node spacing, mesh units")
    ap.add_argument("--padding", type=int, default=1, help="cells between the mesh's box and the lattice's faces (at least 1)")
    ap.add_argument("--exact-band", type=int, default=1, help="cells around each triangle with exact distances (0..8)")
    args = ap.parse_args(argv)
    try:
        m = mesh.read_obj(args.obj)
        ls = mesh.levelset(m, args.h, args.padding, args.exact_band)
    except (OSError, ValueError) as e:
        ap.error(str(e))
    sdf.write(ls, args.sdf)
    print(f"{args.sdf}: {ls.n[0]} x {ls.n[1]} x {ls.n[2]} nodes, h {ls.h:.9g}, origin {' '.join('%.9g' % v for v in ls.header.min)}")
    return 0


def main(argv=None):
    argv = sys.argv[1:] if argv is None else list(argv)
    if argv and argv[0] == "mesh2sdf":
        return mesh2sdf(argv[1:])
    ap = argparse.ArgumentParser(prog="python -m claymore_b200", description="Run a scene and write its frames as .bgeo files.")
    ap.add_argument("-f", "--file", required=True, help="scene JSON (the reference's schema)")
    ap.add_argument("--out", default=".", help="directory of the .bgeo files")
    ap.add_argument("--attributes", default="", help="comma-separated per-particle attributes: v, J")
    ap.add_argument("--resume", default=None, help="checkpoint of this scene to continue from")
    ap.add_argument("--forces", action="store_true", help="write the mean force and torque on each collision body per frame to DIR/forces.csv")
    args = ap.parse_args(argv)
    attributes = [a for a in args.attributes.split(",") if a]
    for a in attributes:
        if a not in ("v", "J"):
            ap.error(f"unknown attribute {a!r} (known: v, J)")
    if not os.path.isdir(args.out):
        ap.error(f"output directory {args.out!r} does not exist")
    sim = parse_scene(args.file, resume=args.resume, forces=args.forces)
    on_frame, fh = None, None
    try:
        if args.forces:
            on_frame, fh = force_recorder(sim, os.path.join(args.out, "forces.csv"), append=args.resume is not None)
        sim.main_loop(on_frame=on_frame, output=args.out, attributes=attributes)
        err = sim.stats().error
    finally:
        if fh is not None:
            fh.close()
        sim.close()
    if err:
        print(f"simulation stopped with error bits {err}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
