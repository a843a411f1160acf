"""Build the UNMODIFIED reference CUDA extensions into oracle/_ref/ (test infrastructure only).

The sources are compiled where they lie (SD_REFERENCE_ROOT; nothing is copied into this repo);
outputs go only to oracle/_ref/, which is git-ignored.
Two torch extensions are produced for sm_90a:

  oracle/_ref/ref_voxlib/ref_voxlib.so            <- imaginaire/model_utils/gancraft/voxlib/*.{cpp,cu}
  oracle/_ref/ref_gridencoder/ref_gridencoder.so  <- gridencoder/src/{gridencoder.cu,bindings.cpp}

and the reference's own Python (the `imaginaire` and `gridencoder` packages, `encoding.py`, `activation.py`,
`configs/`) is STAGED, unmodified, into

  oracle/_ref/py/                                 <- *.py / *.yaml only (about 1 MB)

so that a GPU machine without the reference's sources can import the real
`imaginaire.generators.scenedreamer.Generator` (oracle/refgen.py) when oracle/_ref/ is copied there with the tree.
oracle/_ref/ is git-ignored: nothing of the reference enters this repository's history.

They are used ONLY by tests and by the "reference CUDA" baseline leg of bench.py as the thing we compare
against, never by the product path.  Skips silently when the reference's sources are absent (prebuilt files, if any, are used).
"""
import os
import sys

REF = os.environ.get("SD_REFERENCE_ROOT", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")


def stage_python():
    """Copy the reference's Python sources (unmodified) to oracle/_ref/py/."""
    import shutil
    dst_root = os.path.join(OUT, "py")
    n = 0
    for sub in ("imaginaire", "gridencoder", "configs"):
        for dirpath, dirnames, filenames in os.walk(os.path.join(REF, sub)):
            dirnames[:] = [d for d in dirnames if d not in ("__pycache__", "build", "src")]
            rel = os.path.relpath(dirpath, REF)
            for f in filenames:
                if f.endswith((".py", ".yaml", ".yml", ".csv", ".json", ".txt")):
                    os.makedirs(os.path.join(dst_root, rel), exist_ok=True)
                    shutil.copyfile(os.path.join(dirpath, f), os.path.join(dst_root, rel, f))
                    n += 1
    for f in ("encoding.py", "activation.py", "inference.py", "train.py"):
        if os.path.exists(os.path.join(REF, f)):
            shutil.copyfile(os.path.join(REF, f), os.path.join(dst_root, f))
            n += 1
    print("[oracle/build_ref] staged %d reference files into %s" % (n, dst_root))
    return dst_root


def build(verbose=False):
    if not os.path.isdir(REF):
        print("[oracle/build_ref] %s absent: nothing to build" % REF)
        return False
    stage_python()
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load
    vox = os.path.join(REF, "imaginaire/model_utils/gancraft/voxlib")
    ge = os.path.join(REF, "gridencoder/src")
    jobs = [
        ("ref_voxlib", [os.path.join(vox, f) for f in (
            "voxlib.cpp", "ray_voxel_intersection.cu", "sp_trilinear_worldcoord_kernel.cu",
            "positional_encoding_kernel.cu")], []),
        ("ref_gridencoder", [os.path.join(ge, f) for f in ("gridencoder.cu", "bindings.cpp")],
         ["-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__", "-U__CUDA_NO_HALF2_OPERATORS__"]),
    ]
    for name, srcs, cu_flags in jobs:
        bdir = os.path.join(OUT, name)
        os.makedirs(bdir, exist_ok=True)
        if os.path.exists(os.path.join(bdir, name + ".so")):
            print("[oracle/build_ref] %s already built" % name)
            continue
        load(name=name, sources=srcs, build_directory=bdir, verbose=verbose,
             extra_cflags=["-O3", "-std=c++17"],
             extra_cuda_cflags=["-O3", "-std=c++17", "-lineinfo"] + cu_flags,
             is_python_module=False)
        print("[oracle/build_ref] built", name)
    return True


if __name__ == "__main__":
    build(verbose="-v" in sys.argv)
