"""Build libsmcb.so (hand-written sm_90a CUDA + C-ABI) in-tree with nvcc.

    python -m particles_b200.build

The .so is a git-ignored build product.  nvcc cross-compiles without a GPU.
-fmad=false keeps the few user-level a*b+c of the model maps
un-contracted so that algebraic results (x' = loc + scale*z) are bit-identical to
NumPy's; the CUDA math library (exp/log/sincospi) is unaffected by that flag.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libsmcb.so")
SOURCES = ["smcb_api.cu", "smcb_filter.cu", "smcb_filter_1d.cu", "smcb_filter_nd.cu", "smcb_sampler.cu",
           "smcb_smooth.cu", "smcb_online.cu", "smcb_variance.cu", "smcb_batch.cu", "smcb_bank.cu", "smcb_pmcmc.cu",
           "smcb_nested.cu", "smcb_binary.cu", "smcb_twofilter.cu", "smcb_hmm.cu",
           "smcb_kalman.cu", "smcb_dists.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]      # H100 (Hopper)
NVCC_FLAGS = GENCODE + [
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false", "-Xcompiler", "-fPIC", "--use_fast_math=false",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


STAMP = SO + ".srchash"


def _deps():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h", ".inc"))) + [
        os.path.join(HERE, "..", "include", "smcb.h")]


def source_hash():
    """Content hash of everything the library is compiled from (+ the flags): the stamp written next to the .so."""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for d in _deps():
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def needs_build():
    """Stale if the .so is missing, if the content stamp written by the last build differs from the sources (an edit
    made WHILE a build was running leaves the .so newer than the file it no longer matches), or -- without a stamp --
    if any source is newer than the .so."""
    if not os.path.exists(SO):
        return True
    if os.path.exists(STAMP):
        return open(STAMP).read().strip() != source_hash()
    t = os.path.getmtime(SO)
    return any(os.path.getmtime(d) > t for d in _deps())


def build(force=False, verbose=False, extra=None, out=None):
    """``extra`` (or env SMCB_NVCC_EXTRA, space separated) appends compile flags, e.g. "-DSMCB_SPECULATE=0";
    ``out`` (or env SMCB_BUILD_OUT) names the library to write -- a FULL kernel-variant build next to the
    default one (select it with SMCB_LIB=<out>); the default library is untouched."""
    extra = extra if extra is not None else os.environ.get("SMCB_NVCC_EXTRA", "").split()
    out = out or os.environ.get("SMCB_BUILD_OUT") or SO
    variant = bool(extra) or os.path.abspath(out) != os.path.abspath(SO)
    if not variant and not force and not needs_build():
        return SO
    nvcc = _nvcc()
    stamp = source_hash()                 # of the sources as they are NOW, before the compilers read them
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"] + list(extra)
    tag = ".variant" if variant else ""
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    from concurrent.futures import ThreadPoolExecutor

    def compile_one(src):
        obj = os.path.join(CSRC, src.replace(".cu", tag + ".o"))
        cmd = [nvcc] + flags + (["-Xptxas", "-v"] if verbose else []) + [
            "-c", os.path.join(CSRC, src), "-o", obj]
        subprocess.check_call(cmd)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as pool:      # translation units in parallel
        objs = list(pool.map(compile_one, SOURCES))
    subprocess.check_call([nvcc] + GENCODE + ["-shared", "-o", out]
                          + objs + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    if not variant:
        with open(STAMP, "w") as f:
            f.write(stamp + "\n")
    return out


if __name__ == "__main__":
    if "--stamp" in sys.argv:             # declare the existing .so current (it was built from exactly these sources)
        with open(STAMP, "w") as f:
            f.write(source_hash() + "\n")
        print(STAMP)
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
