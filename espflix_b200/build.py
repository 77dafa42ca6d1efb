"""espflix_b200/build.py — in-tree builds (no JIT cache): the CUDA library, the synthetic stream
generator and the CPU checkers under oracle/. nvcc cross-compiles sm_90a (H100) without a GPU."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "espflix_b200")
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libespflix_b200.so")
SYNTH_LIB = os.path.join(PKG, "synth", "libefsynth.so")
HOST_LIB = os.path.join(PKG, "host", "libespflix_host.so")
HOST_CLI = os.path.join(PKG, "host", "ef_player_cli")
INDEXER_CLI = os.path.join(PKG, "host", "ef_indexer_cli")
ORACLE_LIB = os.path.join(ROOT, "oracle", "libef_oracle.so")
REF_DECODE = os.path.join(ROOT, "oracle", "_ref", "efref_decode")
REF_VIDEO = os.path.join(ROOT, "oracle", "_ref", "libefref_vid.so")

CUDA_SOURCES = ["ef_capi.cu", "ef_decode.cu", "ef_index.cu", "ef_composite.cu", "ef_tsindex.cu", "ef_audio.cu", "ef_library.cu", "ef_trick.cu", "ef_encode.cu", "ef_audio_encode.cu", "ef_idct_tc.cu", "ef_tables.cpp"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources if os.path.exists(s))


def _run(cmd, cwd=None):
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout[-4000:], r.stderr[-4000:]))
    return r


def nvcc_path():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build_cuda(force=False, verbose_ptxas=False):
    srcs = [os.path.join(CSRC, s) for s in CUDA_SOURCES]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(ROOT, "include", "espflix_b200.h"))
    if force or _newer(LIB, deps):
        flags = list(NVCC_FLAGS) + (["-Xptxas", "-v"] if verbose_ptxas else []) + os.environ.get("EF_NVCC_DEFS", "").split()   # tuning experiments
        r = _run([nvcc_path()] + flags + ["-o", LIB] + srcs, cwd=CSRC)
        return r.stderr
    return ""


def build_variant(tag, defs):
    """Tuning variant of the CUDA library with extra nvcc definitions: espflix_b200/libespflix_b200.<tag>.so
    (selected at run time with EF_LIB). Used by tools/sweep_variants.py; never the product."""
    srcs = [os.path.join(CSRC, s) for s in CUDA_SOURCES]
    out = os.path.join(PKG, "libespflix_b200.%s.so" % tag)
    _run([nvcc_path()] + list(NVCC_FLAGS) + defs.split() + ["-o", out] + srcs, cwd=CSRC)
    return out


def build_synth(force=False):
    src = os.path.join(PKG, "synth", "efsynth.cpp")
    if force or _newer(SYNTH_LIB, [src, os.path.join(CSRC, "ef_iso11172_tables.h")]):
        _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", SYNTH_LIB, src])


def build_host(force=False):
    hdir = os.path.join(PKG, "host")
    srcs = [os.path.join(hdir, f) for f in ("player_gpu.cpp", "video_gpu.cpp", "indexer_gpu.cpp")]
    if not all(os.path.exists(s) for s in srcs):
        return
    deps = srcs + [os.path.join(hdir, f) for f in os.listdir(hdir) if f.endswith(".h") or f.endswith("_cli.cpp")]
    if force or _newer(HOST_LIB, deps + [LIB]) or _newer(INDEXER_CLI, deps + [LIB]) or _newer(HOST_CLI, deps + [LIB]):
        common = ["-O2", "-std=c++17", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", hdir]
        link = ["-L", PKG, "-lespflix_b200", "-lpthread"]
        _run(["g++"] + common + ["-shared", "-o", HOST_LIB] + srcs + link + ["-Wl,-rpath,$ORIGIN/.."])
        _run(["g++"] + common + ["-o", HOST_CLI, os.path.join(hdir, "ef_player_cli.cpp")] + srcs + link + ["-Wl,-rpath,$ORIGIN/.."])
        _run(["g++"] + common + ["-o", INDEXER_CLI, os.path.join(hdir, "ef_indexer_cli.cpp")] + srcs + link + ["-Wl,-rpath,$ORIGIN/.."])


def build_oracle(force=False):
    """The checkers: our C restatement always; the unmodified reference too when EF_REFERENCE names a checkout
    of it (tests compare against pins taken from it under tests/golden/ and do not need it). Building the
    checker is not using it."""
    odir = os.path.join(ROOT, "oracle")
    if force:
        _run(["make", "-C", odir, "clean"])
    _run(["make", "-C", odir, "port"])
    ref = os.environ.get("EF_REFERENCE", "")
    if ref and os.path.isdir(os.path.join(ref, "src")):
        _run(["make", "-C", odir, "ref", "REF=" + os.path.abspath(ref)])


def build_all(force=False):
    build_cuda(force)
    build_synth(force)
    build_host(force)
    build_oracle(False)
