"""In-tree build of libuhdr_b200.so: nvcc compiles every translation unit for sm_90a (H100).
Used by __graft_entry__.build(); the .so stays next to this file, importable from the source tree."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libuhdr_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
         # reference CPU path is SSE2 scalar without FMA: keep every float op separately rounded
         "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
         "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden,-O2,-Wall",
         "-I", os.path.join(HERE, "..", "include")]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))


STAMP = OUT + ".stamp"


def source_digest():
    """content hash of everything the library is built from (mtimes do not survive a copy of the tree)"""
    import hashlib
    h = hashlib.sha256()
    deps = sources() + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh")) \
        + glob.glob(os.path.join(CSRC, "*.inc")) + glob.glob(os.path.join(HERE, "..", "include", "*.h")) \
        + glob.glob(os.path.join(HERE, "..", "include", "*.hpp")) + [os.path.abspath(__file__)]
    for d in sorted(deps):
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def needs_build():
    if not os.path.exists(OUT) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        return f.read().strip() != source_digest()


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs, procs = [], []
    for s in sources():
        o = os.path.join(objdir, os.path.basename(s) + ".o")
        objs.append(o)
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-x", "cu", "-c", s, "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    ok = True
    for s, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {os.path.basename(s)}\n{out}\n")
        ok &= p.returncode == 0
    if not ok:
        raise RuntimeError("nvcc failed")
    # link next to the target and swap it in atomically: a process loading the library during a build sees
    # either the previous library or the new one, never a half-written file
    tmp = OUT + ".link"
    subprocess.check_call([NVCC] + ARCH + ["-shared", "-o", tmp] + objs + ["-lcudart", "-lpthread"])
    os.replace(tmp, OUT)
    with open(STAMP + ".tmp", "w") as f:
        f.write(source_digest())
    os.replace(STAMP + ".tmp", STAMP)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
