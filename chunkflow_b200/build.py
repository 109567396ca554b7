"""Build the native library IN-TREE with nvcc for sm_90a (cross-compiles without a GPU).

    python -m chunkflow_b200.build [--force]

Output: chunkflow_b200/_native/libchunkflow_b200.so (git-ignored).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_native")
LIB_PATH = os.path.join(OUT_DIR, "libchunkflow_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


HASH_PATH = LIB_PATH + ".srchash"


def _source_hash() -> str:
    """sha256 over the native sources, the header and the compiler flags (file copies do not always keep mtimes)."""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    deps = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(ROOT, "include", "chunkflow_b200.h")]
    for d in deps:
        if not os.path.isfile(d):
            continue
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    try:
        with open(HASH_PATH) as f:
            return f.read().strip() != _source_hash()
    except OSError:
        return True


def build_variant(name: str, defines) -> str:
    """Development build with extra -D flags into _native/libchunkflow_b200_<name>.so (load it with CFB_NATIVE_LIB)."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    out = os.path.join(OUT_DIR, f"libchunkflow_b200_{name}.so")
    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = [nvcc, *NVCC_FLAGS, *defines, "-I", os.path.join(ROOT, "include"), "-I", CSRC, *sources(), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return out


def build_native(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB_PATH
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libchunkflow_b200.so")
    os.makedirs(OUT_DIR, exist_ok=True)
    extra = os.environ.get("CFB_NVCC_DEFINES", "").split()  # development builds only, e.g. -DCFB_TS_TRACE
    cmd = [nvcc, *NVCC_FLAGS, *extra, "-I", os.path.join(ROOT, "include"), "-I", CSRC, *sources(), "-o", LIB_PATH]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd))
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stdout + res.stderr)
    if not extra:  # a build with development defines must not pass for the product library
        with open(HASH_PATH, "w") as f:
            f.write(_source_hash())
    elif os.path.exists(HASH_PATH):
        os.remove(HASH_PATH)
    return LIB_PATH


if __name__ == "__main__":
    if "--variant" in sys.argv:  # python -m chunkflow_b200.build --variant trace -DCFB_TS_TRACE
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], sys.argv[i + 2:]))
        sys.exit(0)
    print(build_native(force="--force" in sys.argv, verbose="-v" in sys.argv))
