"""In-tree build of the native extension ``bee2bee_b200/_C*.so`` for sm_90a (H100).

Plain ``nvcc`` for the kernel translation units (no torch headers -> seconds each),
``g++`` for the single torch-facing binding, one link step.  Objects are cached by a
content hash under ``build/`` so repeated ``build()`` calls are incremental.  The
resulting ``.so`` lives inside the package, so the tree is importable as built (no JIT cache
under ``~/.cache``).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "csrc"
BUILD = ROOT / "build" / "obj"
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")

CU_SOURCES = ["gemm_tc.cu", "elementwise.cu", "attention.cu", "attention_tc.cu", "sampler.cu"]
CPP_SOURCES = ["peer.cpp", "binding.cpp"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--use_fast_math", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


def ext_path() -> Path:
    suffix = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return ROOT / "bee2bee_b200" / f"_C{suffix}"


def _hash(paths, extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for p in paths:
        h.update(Path(p).read_bytes())
    return h.hexdigest()[:16]


def _run(cmd, log: Path | None = None) -> None:
    res = subprocess.run(cmd, capture_output=True, text=True)
    if log is not None:
        log.write_text(res.stdout + res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("build step failed: " + " ".join(map(str, cmd)))


def build(verbose: bool = True, force: bool = False) -> Path:
    import torch
    from torch.utils import cpp_extension as ce

    BUILD.mkdir(parents=True, exist_ok=True)
    headers = sorted(CSRC.glob("*.h")) + sorted(CSRC.glob("*.cuh"))
    inc = [f"-I{p}" for p in ce.include_paths()] + [f"-I{CUDA_HOME}/include", f"-I{sysconfig.get_paths()['include']}"]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx_flags = ["-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_EXTENSION_NAME=_C",
                 "-DTORCH_API_INCLUDE_EXTENSION_H", "-w"]

    jobs = []
    objs = []
    for src in CU_SOURCES:
        s = CSRC / src
        tag = _hash([s] + headers, " ".join(NVCC_FLAGS))
        obj = BUILD / f"{s.stem}.{tag}.o"
        objs.append(obj)
        if force or not obj.exists():
            jobs.append(([NVCC, *NVCC_FLAGS, f"-I{CSRC}", "-c", str(s), "-o", str(obj)], BUILD / f"{s.stem}.ptxas.log"))
    for src in CPP_SOURCES:
        s = CSRC / src
        tag = _hash([s] + headers, " ".join(cxx_flags) + torch.__version__)
        obj = BUILD / f"{s.stem}.{tag}.o"
        objs.append(obj)
        if force or not obj.exists():
            jobs.append((["g++", *cxx_flags, *inc, f"-I{CSRC}", "-c", str(s), "-o", str(obj)], None))

    # drop objects of older source revisions (the cache is keyed by content hash)
    keep = {o.name for o in objs}
    for old in BUILD.glob("*.o"):
        if old.name not in keep:
            old.unlink(missing_ok=True)

    if jobs:
        if verbose:
            print(f"[bee2bee_b200] compiling {len(jobs)} translation unit(s) for sm_90a ...", flush=True)
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda j: _run(*j), jobs))

    out = ext_path()
    link_tag = _hash(objs, "link")
    stamp = BUILD / "link.stamp"
    if force or jobs or not out.exists() or not stamp.exists() or stamp.read_text() != link_tag:
        libdirs = ce.library_paths(device_type="cuda") if "device_type" in ce.library_paths.__code__.co_varnames else ce.library_paths(True)
        ld = [f"-L{p}" for p in libdirs] + [f"-L{CUDA_HOME}/lib64"]
        rpath = [f"-Wl,-rpath,{p}" for p in libdirs]
        libs = ["-lc10", "-ltorch_cpu", "-ltorch", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart"]
        _run(["g++", "-shared", *map(str, objs), *ld, *rpath, *libs, "-o", str(out)])
        stamp.write_text(link_tag)
        if verbose:
            print(f"[bee2bee_b200] linked {out}", flush=True)
    return out


if __name__ == "__main__":
    build(force="--force" in sys.argv)
