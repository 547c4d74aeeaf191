"""Builds htslib_b200/libhtsgpu.so in-tree with nvcc for sm_90a (no torch involved)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, os.environ.get("HGPU_OUT", "libhtsgpu.so"))      # HGPU_OUT: side-by-side tuning builds
BUILD = os.path.join(HERE, os.environ.get("HGPU_BUILD_DIR", "build"))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "--use_fast_math", "-Xptxas", "-v"]
FLAGS += os.environ.get("HGPU_DEFS", "").split()
if os.environ.get("HGPU_PROFILE"):
    FLAGS.append("-DHGPU_PROFILE")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    deps.append(os.path.join(HERE, "..", "include", "htsgpu.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    os.makedirs(BUILD, exist_ok=True)
    for src in sources():
        obj = os.path.join(BUILD, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [NVCC] + FLAGS + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError("nvcc failed on %s" % src)
    with open(os.path.join(BUILD, "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        sys.stderr.write("\n".join(log))
    cmd = [NVCC, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static", "-lpthread", "-ldl", "-lrt"]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
