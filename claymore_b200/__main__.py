"""The scene runner, the reference's `gmpm -f scene.json` (Projects/GMPM/gmpm.cu):

    python -m claymore_b200 -f scene.json [--out DIR] [--attributes v,J] [--resume CKPT]

parse_scene, then main_loop: every finished frame is written to DIR (default: the working directory) as
model_id[i]_frame[f].bgeo, with the per-particle attributes listed (v: velocity, J: volume ratio).  --resume continues a
checkpoint of the same scene and writes only its remaining frames.
"""
import argparse
import os
import sys

from .scene import parse_scene


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m claymore_b200", description="Run a scene and write its frames as .bgeo files.")
    ap.add_argument("-f", "--file", required=True, help="scene JSON (the reference's schema)")
    ap.add_argument("--out", default=".", help="directory of the .bgeo files")
    ap.add_argument("--attributes", default="", help="comma-separated per-particle attributes: v, J")
    ap.add_argument("--resume", default=None, help="checkpoint of this scene to continue from")
    args = ap.parse_args(argv)
    attributes = [a for a in args.attributes.split(",") if a]
    for a in attributes:
        if a not in ("v", "J"):
            ap.error(f"unknown attribute {a!r} (known: v, J)")
    if not os.path.isdir(args.out):
        ap.error(f"output directory {args.out!r} does not exist")
    sim = parse_scene(args.file, resume=args.resume)
    try:
        sim.main_loop(output=args.out, attributes=attributes)
        err = sim.stats().error
    finally:
        sim.close()
    if err:
        print(f"simulation stopped with error bits {err}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
