"""Build libnerfloam_b200.so (hand-written sm_90a CUDA + host C++) in-tree with nvcc.

    python nerf-loam_b200/build.py            # incremental
    python nerf-loam_b200/build.py --force

The library is plain C ABI (include/nerfloam_b200.h); it links only against the CUDA runtime
(statically), not against torch.  nvcc cross-compiles without a GPU.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libnerfloam_b200.so")
SOURCES = ["nl_error.cpp", "octree_host.cpp", "grid_dropin.cu", "render.cu", "gather.cu", "mlp.cu", "mlp_tc.cu", "pose.cu", "optim.cu", "mc.cu", "peer.cu", "select.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "--extended-lambda", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "nerfloam_b200.h"))
    objs = []
    procs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, os.path.splitext(src)[0] + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [_nvcc()] + ARCH + FLAGS + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd))
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(out.decode())
        elif verbose and out:
            sys.stdout.write(out.decode())
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(LIB, objs):
        cmd = [_nvcc()] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return LIB


SVO_LIB = os.path.join(HERE, "svo_b200.so")


def build_svo_shim(force=False, verbose=False):
    """TorchScript custom-class shim `torch.classes.svo.Octree` (csrc/shim/svo_torch.cpp): host-only C++ compiled with g++
    against libtorch; it carries its own copy of the octree (octree_host.cpp, nl_error.cpp), so it has no CUDA dependency and can
    be loaded with torch.classes.load_library() exactly where the reference loads its svo extension (src/mapping.py:19-20)."""
    from torch.utils import cpp_extension as ce
    import torch
    src = [os.path.join(CSRC, "shim", "svo_torch.cpp"), os.path.join(CSRC, "octree_host.cpp"), os.path.join(CSRC, "nl_error.cpp")]
    deps = src + [os.path.join(os.path.dirname(HERE), "include", "nerfloam_b200.h"), os.path.join(CSRC, "nl_error.h")]
    if not (force or _stale(SVO_LIB, deps)):
        return SVO_LIB
    inc = [a for pth in ce.include_paths() for a in ("-isystem", pth)] + ["-I", os.path.join(os.path.dirname(HERE), "include"), "-I", CSRC]
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", abi, "-DNL_NO_CUDA"] + inc + src + \
          ["-o", SVO_LIB, "-L", libdir, "-Wl,-rpath," + libdir, "-ltorch", "-ltorch_cpu", "-lc10"]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return SVO_LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
    print(build_svo_shim(force="--force" in sys.argv, verbose=True))
