"""Build the UNMODIFIED reference native extensions into oracle/_ref/ (test infrastructure only).

  svo  : /root/reference/third_party/sparse_octree  (C++ TorchScript custom class, CPU)
  grid : /root/reference/third_party/sparse_voxels  (C++ + CUDA, pybind11), compiled for sm_90a

Sources are compiled where they lie under /root/reference (never copied); outputs go only to
oracle/_ref/ (git-ignored, but shipped to the GPU box by gpurun).  The reference's own setup.py is
NOT run; this is a direct torch.utils.cpp_extension.load() of the few source files.
The one missing dependency (Eigen, used for a 3-int return type) is satisfied by oracle/shim/.

The reference's hot-path PYTHON (render_helpers / voxel_helpers / lidar / criterion / se3pose / lidarFrame /
sample_util, ~1500 lines) is *staged* by stage_src() into oracle/_ref/src/ the same way: a build product in the
git-ignored oracle/_ref/ (never committed, never imported by the product) that travels to the GPU box with the
snapshot, so that the GPU tests and bench.py can run the UNMODIFIED reference loop (with grid_ref.so) beside the
product on the same GPU (oracle/ref_harness.py).

Usage:  python oracle/build_ref.py [svo] [grid] [src]
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("NERFLOAM_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref")


def build_svo():
    from torch.utils.cpp_extension import load
    src = os.path.join(REF, "third_party", "sparse_octree", "src")
    bdir = os.path.join(OUT, "svo")
    os.makedirs(bdir, exist_ok=True)
    load(name="svo_ref", sources=[os.path.join(src, "octree.cpp"), os.path.join(src, "bindings.cpp")],
         extra_include_paths=[os.path.join(HERE, "shim")], extra_cflags=["-O2", "-w"],
         build_directory=bdir, is_python_module=False, verbose=False)
    return os.path.join(bdir, "svo_ref.so")


def build_grid():
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    from torch.utils.cpp_extension import load
    src = os.path.join(REF, "third_party", "sparse_voxels", "src")
    bdir = os.path.join(OUT, "grid")
    os.makedirs(bdir, exist_ok=True)
    names = ["binding.cpp", "intersect.cpp", "sample.cpp", "octree.cpp", "intersect_gpu.cu", "sample_gpu.cu"]
    load(name="grid_ref", sources=[os.path.join(src, n) for n in names],
         extra_cflags=["-O2", "-w"], extra_cuda_cflags=["-O2", "-w"],
         build_directory=bdir, is_python_module=True, verbose=False)
    return os.path.join(bdir, "grid_ref.so")


REF_PY = ["criterion.py", "se3pose.py", "lidarFrame.py", "utils/__init__.py", "utils/sample_util.py",
          "variations/render_helpers.py", "variations/voxel_helpers.py", "variations/lidar.py"]


def stage_src():
    """Stage the reference's hot-path Python files, byte for byte, under oracle/_ref/src (git-ignored build product)."""
    import shutil
    dst = os.path.join(OUT, "src")
    for rel in REF_PY:
        s, d = os.path.join(REF, "src", rel), os.path.join(dst, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        shutil.copyfile(s, d)
    return dst


if __name__ == "__main__":
    if not os.path.isdir(REF):
        print("reference tree not present; nothing to build")
        sys.exit(0)
    what = sys.argv[1:] or ["svo", "grid", "src"]
    for w in what:
        p = {"svo": build_svo, "grid": build_grid, "src": stage_src}[w]()
        print("built", p)
