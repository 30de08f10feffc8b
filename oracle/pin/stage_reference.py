"""Stage the original project's Python packages: <reference>/{pyramid_dit,video_vae,diffusion_schedulers,trainer_misc}
(+ the top-level utils.py they import) -> oracle/_ref/ (git-ignored, like the built library).

TEST / BASELINE INFRASTRUCTURE.  <reference> is a checkout of jy0205/Pyramid-Flow: $PYRAMID_FLOW_REFERENCE, or a directory
`reference` next to this repository.  Where it is readable, build() stages it; the drop-in test (tests/test_dropin_gpu.py)
and bench.py's `gpu_eager_baseline` leg import the UNMODIFIED reference from the staged copy through oracle/pin/ref_shim.py,
and skip / report "unavailable" without it.  Nothing is edited: files are copied byte for byte (checked below), never
committed, and no product module imports them.

    python oracle/pin/stage_reference.py        (also run by __graft_entry__.build())
"""
from __future__ import annotations

import filecmp
import os
import shutil
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
SRC = Path(os.environ.get("PYRAMID_FLOW_REFERENCE") or ROOT.parent / "reference")
DST = ROOT / "oracle" / "_ref"
PACKAGES = ("pyramid_dit", "video_vae", "diffusion_schedulers", "trainer_misc")
TOP_FILES = ("utils.py",)          # video_vae/modeling_causal_conv.py:11 imports the context-parallel helpers from it


def source_readable() -> bool:
    try:
        return (SRC / "pyramid_dit").is_dir()
    except OSError:          # e.g. the parent directory is not searchable by this user
        return False


def stage(verbose: bool = True) -> bool:
    if not source_readable():
        if verbose:
            print(f"[stage_reference] {SRC} not readable: using the staged copy at {DST}" if DST.exists()
                  else f"[stage_reference] neither {SRC} nor {DST} exists")
        return DST.exists()
    DST.mkdir(parents=True, exist_ok=True)
    n = 0
    for pkg in PACKAGES:
        for f in (SRC / pkg).rglob("*.py"):
            out = DST / f.relative_to(SRC)
            out.parent.mkdir(parents=True, exist_ok=True)
            if not out.exists() or not filecmp.cmp(f, out, shallow=False):
                shutil.copyfile(f, out)
            n += 1
    for name in TOP_FILES:
        if not (DST / name).exists() or not filecmp.cmp(SRC / name, DST / name, shallow=False):
            shutil.copyfile(SRC / name, DST / name)
        n += 1
    (DST / "STAGED_FROM").write_text(f"{SRC} (unmodified copy of {', '.join(PACKAGES)}; {n} files)\n")
    if verbose:
        print(f"[stage_reference] {n} files -> {DST}")
    return True


if __name__ == "__main__":
    sys.exit(0 if stage() else 1)
