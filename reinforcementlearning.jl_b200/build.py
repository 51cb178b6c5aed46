"""Build libb200rl.so in-tree with nvcc for sm_90a (H100; no torch, no JIT cache).

    python reinforcementlearning.jl_b200/build.py [--force] [--verbose]

Per-file flags: the env and returns kernels must not contract a*b+c (the reference's Julia
code never does), so those translation units get -fmad=false; the NN kernels keep FMA."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200rl.so")
BUILD = os.path.join(HERE, "build")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-diag-suppress", "177"]
# (source, extra flags)
SOURCES = [
    ("core.cu", []),
    ("env.cu", ["-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false"]),
    ("returns.cu", ["-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false"]),
    ("comm.cu", []),
]
ENV_FLAGS = ["-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false"]
OPTIONAL = [("traj.cu", []), ("nn.cu", []), ("algo.cu", []), ("nn_tc.cu", []), ("fwd_tc.cu", ENV_FLAGS)]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def _digest(paths, flags):
    h = hashlib.sha256()
    h.update(" ".join(flags).encode())
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build(force=False, verbose=False, variant=None, defs=()):
    """variant = None: the product library.  variant = "name" (+ defs = ["-DX=1", ...]): an A/B build of the same sources with extra
    defines into build/variants/<name>/libb200rl.so, loaded instead of the product library when B200RL_LIB points at it
    (development only: lets one GPU call time several variants of a kernel on the same box)."""
    out_dir = BUILD if variant is None else os.path.join(BUILD, "variants", variant)
    out_so = OUT if variant is None else os.path.join(out_dir, "libb200rl.so")
    os.makedirs(out_dir, exist_ok=True)
    nvcc = _nvcc()
    env = dict(os.environ)
    # the image exports CC/CXX pointing at a wrapper without libgomp specs; use the system g++
    host_cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    headers = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "b200rl.h"))
    srcs = list(SOURCES) + [(s, f) for s, f in OPTIONAL if os.path.exists(os.path.join(CSRC, s))]
    objs, rebuilt = [], False
    for src, extra in srcs:
        path = os.path.join(CSRC, src)
        obj = os.path.join(out_dir, src.replace(".cu", ".o"))
        stamp = obj + ".sha"
        flags = ARCH + COMMON + extra + list(defs)
        dig = _digest([path] + headers, flags)
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
            continue
        cmd = [nvcc, "-ccbin", host_cxx] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", path, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd, env=env)
        open(stamp, "w").write(dig)
        rebuilt = True
    if rebuilt or not os.path.exists(out_so):
        cmd = [nvcc, "-ccbin", host_cxx] + ARCH + ["-shared", "-Xcompiler", "-fPIC", "-o", out_so] + objs + ["-ldl"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd, env=env)
    return out_so


if __name__ == "__main__":
    if "--variant" in sys.argv:      # python build.py --variant NAME -DFOO=1 -DBAR
        name = sys.argv[sys.argv.index("--variant") + 1]
        print(build(variant=name, defs=[a for a in sys.argv if a.startswith("-D")], verbose="--verbose" in sys.argv))
    else:
        print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
