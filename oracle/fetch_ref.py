"""Copies the reference project's vendored pretrained weights (data, not source) into oracle/_ref/checkpoints/, where
bench.py's I3D / RAFT lines and scripts/precision/ read them; the tests use seeded stand-ins and do not need them.
oracle/_ref/ is git-ignored.  The reference checkout is taken from
$VF_REFERENCE_DIR (default /root/reference, a read-only checkout of the upstream video_features project).  Files that
are already present are kept; when neither the copy nor the reference is there this prints what is missing."""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(os.environ.get("VF_REFERENCE_DIR", "/root/reference"), "models")
DST = os.path.join(ROOT, "oracle", "_ref", "checkpoints")
FILES = ("i3d/checkpoints/i3d_rgb.pt", "i3d/checkpoints/i3d_flow.pt", "raft/checkpoints/raft-sintel.pth")


def main() -> None:
    os.makedirs(DST, exist_ok=True)
    for rel in FILES:
        dst = os.path.join(DST, os.path.basename(rel))
        src = os.path.join(REF, rel)
        if os.path.exists(dst):
            continue
        if os.path.exists(src):
            shutil.copyfile(src, dst)
            print("copied", rel)
        else:
            print(f"fetch_ref: {src} not found; {dst} stays missing", file=sys.stderr)


if __name__ == "__main__":
    main()
