"""In-tree build of the CUDA library for sm_90a (nvcc cross-compiles without a GPU)."""
import hashlib
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIBDIR = os.path.join(_HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIBNAME = "libagentainer_b200.so"
SOURCES = ["agr_kernels.cu", "agr_k1_tma.cu", "agr_k1_var.cu", "agr_k4.cu", "agr_k5_json.cu", "agr_svc.cu", "agr_json_host.cpp", "agr_engine.cu",
           "agr_front.cu", "agr_snapshot.cu", "agr_exchange.cu", "agr_relayout.cu"]
HEADERS = ["agr_common.h", "agr_agents.hpp", "agr_synth.h", "agr_kernels.cuh", "agr_device.cuh", "agr_svc.h", "agr_ring.hpp", "agr_engine.h",
           os.path.join("..", "..", "include", "agentainer_gpu.h")]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100 (Hopper): TMA, mbarrier
NVCC_FLAGS = GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def lib_path() -> str:
    return os.path.join(LIBDIR, LIBNAME)


def source_hash() -> str:
    """sha256 over every source, header and the compiler flags: what the built library is a function of."""
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for f in SOURCES + HEADERS:
        p = os.path.join(CSRC, f)
        if os.path.exists(p):
            h.update(f.encode()); h.update(open(p, "rb").read())
    return h.hexdigest()


def _stamp_path() -> str:
    return lib_path() + ".srchash"


def _stale() -> bool:
    """The library is stale when it is missing or was built from other sources than the ones in the tree (content hash, not
    mtime: a checkout or a copy to another machine changes mtimes but not what the binary was compiled from)."""
    if not os.path.exists(lib_path()) or not os.path.exists(_stamp_path()):
        return True
    return open(_stamp_path()).read().strip() != source_hash()


def build_native(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/* into lib/libagentainer_b200.so (one nvcc per translation unit, in parallel, then one link)."""
    if not force and not _stale():
        return lib_path()
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libagentainer_b200.so (and there is no CPU fallback)")
    os.makedirs(OBJDIR, exist_ok=True)

    def compile_one(src: str):
        obj = os.path.join(OBJDIR, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas=-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        res = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, res

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        results = list(ex.map(compile_one, SOURCES))
    for src, _, res in results:
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n" + res.stdout + res.stderr)
        if verbose:
            print(res.stderr)
    cmd = [nvcc] + GENCODE + ["-shared", "-Xcompiler", "-fPIC"] + [o for _, o, _ in results] + [
        "-o", lib_path(), "-lcudart", "-ldl", "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
    with open(_stamp_path(), "w") as f:
        f.write(source_hash() + "\n")
    return lib_path()


HOST = os.path.join(_HERE, "host")


def _gxx(srcs, out, force):
    deps = srcs + [os.path.join(HOST, "requests.hpp"), os.path.join(_HERE, "..", "include", "agentainer_gpu.h"), lib_path()]
    if not force and os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps if os.path.exists(d)):
        return out
    gxx = shutil.which("g++")
    if not gxx:
        raise RuntimeError("g++ not found")
    cmd = [gxx, "-O2", "-std=c++17", "-Wall", "-I" + os.path.join(_HERE, "..", "include")] + srcs + [
        "-o", out, "-L" + LIBDIR, "-lagentainer_b200", "-Wl,-rpath,$ORIGIN/../lib", "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed:\n" + res.stdout + res.stderr)
    return out


def build_host(force: bool = False) -> str:
    """Compile the C++ mirror of requests.Manager / ReplayWorker with its threaded driver (host/test_host) and the
    single-request caller benchmark (host/bench_callers)."""
    _gxx([os.path.join(HOST, "bench_callers.cpp")], os.path.join(HOST, "bench_callers"), force)
    return _gxx([os.path.join(HOST, f) for f in ("requests.cpp", "test_host.cpp")], os.path.join(HOST, "test_host"), force)
