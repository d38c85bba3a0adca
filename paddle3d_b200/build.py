"""Build libp3d_b200.so in-tree with nvcc for sm_90a (one object per .cu, in parallel)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(HERE, "libp3d_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]  # Hopper (H100): wgmma, TMA
FLAGS = ["-O3", "-std=c++17"] + ARCH + ["-lineinfo", "-Xcompiler", "-fPIC",
         "-I", os.path.join(ROOT, "include"), "-I", CSRC] + os.environ.get("P3D_NVCC_EXTRA", "").split()


def _newer(src, dst, deps):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(p) > t for p in [src] + deps)


def build(verbose=False, force=False, out_dir=None, extra_flags=()):
    """out_dir / extra_flags: build a variant (e.g. -DP3D_DENSE_TRACE) into another directory; the in-tree library is
    the default."""
    obj_dir = os.path.join(out_dir, "_obj") if out_dir else OBJ
    lib_path = os.path.join(out_dir, "libp3d_b200.so") if out_dir else LIB
    os.makedirs(obj_dir, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + \
           [os.path.join(ROOT, "include", "p3d_b200.h")]
    jobs = []
    for s in srcs:
        src, obj = os.path.join(CSRC, s), os.path.join(obj_dir, s[:-3] + ".o")
        if force or _newer(src, obj, hdrs):
            jobs.append((src, obj))

    def cc(job):
        cmd = [NVCC] + FLAGS + list(extra_flags) + (["-Xptxas", "-v"] if verbose else []) + ["-c", job[0], "-o", job[1]]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return job[0], r.returncode, r.stdout + r.stderr

    failed = False
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for src, rc, out in ex.map(cc, jobs):
            if rc != 0 or verbose:
                sys.stderr.write("== %s\n%s\n" % (src, out))
            failed |= rc != 0
    if failed:
        raise RuntimeError("nvcc failed")
    objs = [os.path.join(obj_dir, s[:-3] + ".o") for s in srcs]
    if jobs or not os.path.exists(lib_path):
        cmd = [NVCC, "-shared"] + ARCH + ["-o", lib_path] + objs
        subprocess.run(cmd, check=True)
    return lib_path


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
