"""In-tree builds of libnqb.so and of the per-signature kernel libraries (sm_90a only).

``nvcc -gencode arch=compute_90a,code=sm_90a`` cross-compiles without a GPU, so
``__graft_entry__.build()`` can run on a machine without one; the resulting ``.so`` files
are loaded from the tree on the H100.  At run time a signature that has no
prebuilt library is generated and compiled on the spot (the same thing the
reference's OpenEquivariance backend does with its JIT, nequip/nn/_tp_scatter_oeq.py:29-47);
if ``nvcc`` is missing that is a hard error -- there is no CPU fallback.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import threading
from concurrent.futures import ThreadPoolExecutor
from typing import Iterable, List, Optional, Tuple

from .codegen import CODEGEN_VERSION, GenOptions, TPSignature, generate

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIBDIR = os.path.join(_HERE, "lib")
GENDIR = os.path.join(_HERE, "_gen")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON_FLAGS = ["-O3", "-lineinfo", "-std=c++17", "-shared", "-Xcompiler", "-fPIC"]

_lock = threading.Lock()


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError(
            "nequip_b200: nvcc not found -- the H100 kernels cannot be built and there is no CPU fallback"
        )
    return p


def _run(cmd: List[str]):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nequip_b200 build failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return r.stdout + r.stderr


def _newer(src_files: Iterable[str], target: str) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_files)


def runtime_lib_path() -> str:
    return os.path.join(LIBDIR, "libnqb.so")


def ensure_runtime(force: bool = False) -> str:
    """Build (if stale) and return the path of libnqb.so."""
    out = runtime_lib_path()
    cus = [os.path.join(CSRC, n) for n in ("nqb_runtime.cu", "nqb_mlp.cu", "nqb_gemm.cu", "nqb_nl.cu",
                                             "nqb_pair.cu", "nqb_md.cu", "nqb_relax.cu", "nqb_npt.cu")]
    srcs = cus + [os.path.join(INCLUDE, "nqb.h"), os.path.join(CSRC, "nqb_tc.cuh")]
    with _lock:
        if force or _newer(srcs, out):
            os.makedirs(LIBDIR, exist_ok=True)
            tmp = out + f".tmp{os.getpid()}"
            _run([nvcc_path(), *ARCH_FLAGS, *COMMON_FLAGS, "-I", INCLUDE, "-Xptxas", "-v", "-o", tmp, *cus, "-ldl"])
            os.replace(tmp, out)
    return out


def _device_header_hash() -> str:
    """Hash of the headers every generated kernel library includes (part of its file name)."""
    h = hashlib.sha1()
    for name in ("nqb_tc.cuh", "nqb_tp_device.cuh", "nqb_tp_fused.cuh"):
        with open(os.path.join(CSRC, name), "rb") as f:
            h.update(f.read())
    return h.hexdigest()[:8]


def spec_lib_path(sig: TPSignature, opts: Optional[GenOptions] = None) -> str:
    opts = opts or GenOptions()
    return os.path.join(LIBDIR, f"nqbspec_{sig.key(opts)}_{_device_header_hash()}.so")


def ensure_spec(sig: TPSignature, opts: Optional[GenOptions] = None) -> str:
    """Generate + compile the kernel library of one signature (cached in-tree)."""
    out = spec_lib_path(sig, opts)
    if os.path.exists(out):
        return out
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(GENDIR, exist_ok=True)
    # several processes (ranks) or threads may build the same signature at once: each writes its own source and
    # temporary library, and the final renames are atomic
    stem = os.path.join(GENDIR, os.path.basename(out)[:-3])
    uniq = f"{os.getpid()}_{threading.get_ident()}"
    cu, tmp = f"{stem}.{uniq}.cu", f"{out}.tmp{uniq}"
    with open(cu, "w") as f:
        f.write(generate(sig, opts))
    _run([nvcc_path(), *ARCH_FLAGS, *COMMON_FLAGS, "-I", CSRC, "-o", tmp, cu])
    os.replace(tmp, out)
    os.replace(cu, stem + ".cu")
    return out


def ensure_specs(sigs: Iterable[Tuple[TPSignature, Optional[GenOptions]]], jobs: int = 0) -> List[str]:
    """Parallel build of many signatures (used by __graft_entry__.build)."""
    jobs = jobs or min(8, os.cpu_count() or 1)
    with ThreadPoolExecutor(max_workers=jobs) as ex:
        return list(ex.map(lambda item: ensure_spec(*item), sigs))


__all__ = [
    "ensure_runtime",
    "ensure_spec",
    "ensure_specs",
    "spec_lib_path",
    "runtime_lib_path",
    "CODEGEN_VERSION",
]
