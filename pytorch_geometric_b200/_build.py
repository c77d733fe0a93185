"""In-tree build of libb200mp.so (the C-ABI library) with nvcc for sm_90a (H100).

No torch involvement: the library only depends on the CUDA runtime (statically linked), so the
same .so serves Python (ctypes), C, C++ or any FFI.  The .so lands in pytorch_geometric_b200/lib/ next to
a stamp file holding the SHA-256 of every source, header and compiler flag it was built from (both are
git-ignored).  Staleness is decided by that fingerprint, NOT by file times: a copied tree does not keep
mtimes in any useful order, and a spurious rebuild costs minutes of nvcc.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.environ.get("B200MP_OBJ_DIR", os.path.join("/tmp", f"b200mp_build_{os.getuid()}"))  # objects stay out of tree
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libb200mp.so")
STAMP = os.path.join(LIBDIR, "libb200mp.sha256")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *ARCH_FLAGS, "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
    "-Wno-deprecated-declarations", "-DB200MP_BUILD",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found: the b200mp CUDA library cannot be built")
    return cand


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(INCLUDE, "b200mp.h"))
    return sorted(hs)


def _digest(*paths, extra: str = "") -> str:
    h = hashlib.sha256((" ".join(NVCC_FLAGS) + extra).encode())
    for path in paths:
        h.update(os.path.basename(path).encode())
        with open(path, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def fingerprint() -> str:
    """SHA-256 over the compiler flags and the contents of every source and header."""
    return _digest(*(sources() + _headers()))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    try:
        with open(STAMP) as fh:
            return fh.read().strip() != fingerprint()
    except OSError:
        return True


def _private_obj_dir() -> str:
    """Object cache owned by this user with mode 0700 (a pre-created, foreign or world-writable directory is
    refused: objects found there would be linked into the library)."""
    os.makedirs(OBJ, mode=0o700, exist_ok=True)
    st = os.stat(OBJ)
    if st.st_uid != os.getuid() or (st.st_mode & 0o022):
        raise RuntimeError(f"object directory {OBJ} is not owned by uid {os.getuid()} or is writable by others; "
                           "set B200MP_OBJ_DIR to a directory you own (mode 0700)")
    if st.st_mode & 0o077:
        os.chmod(OBJ, 0o700)
    return OBJ


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    import fcntl
    obj_dir = _private_obj_dir()
    os.makedirs(LIBDIR, exist_ok=True)
    nvcc = _nvcc()
    hdr_digest = _digest(*_headers())
    # one builder at a time (ranks of one job race for the same files); late comers re-check the stamp
    with open(os.path.join(obj_dir, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not needs_build():
            return LIB

        def compile_one(src):
            # objects are keyed by the content of the source, of every header and by the flags: a snapshot copy,
            # a touched file or a changed flag can never link a stale object
            key = _digest(src, extra=hdr_digest)[:24]
            obj = os.path.join(obj_dir, f"{os.path.basename(src)[:-3]}.{key}.o")
            if not force and os.path.exists(obj):
                return obj
            tmp = f"{obj}.{os.getpid()}.tmp"
            cmd = [nvcc, *NVCC_FLAGS, "-I", INCLUDE, "-c", src, "-o", tmp]
            if verbose:
                print(" ".join(cmd), file=sys.stderr)
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
            os.replace(tmp, obj)
            return obj

        with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 4)) as ex:
            objs = list(ex.map(compile_one, sources()))
        tmp_lib = f"{LIB}.{os.getpid()}.tmp"
        cmd = [nvcc, "-shared", *ARCH_FLAGS, "-o", tmp_lib, *objs,
               "-Xlinker", "--exclude-libs,ALL"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        os.replace(tmp_lib, LIB)                         # atomic: a concurrent dlopen sees the old or the new file
        with open(STAMP + ".tmp", "w") as fh:
            fh.write(fingerprint() + "\n")
        os.replace(STAMP + ".tmp", STAMP)
        # drop objects of older source revisions
        keep = set(objs)
        for f in os.listdir(obj_dir):
            path = os.path.join(obj_dir, f)
            if f.endswith(".o") and path not in keep:
                try:
                    os.unlink(path)
                except OSError:
                    pass
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
