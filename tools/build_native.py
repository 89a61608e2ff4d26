"""Build the native module in-tree: infinistore_b200/_infinistore*.so.

g++ (C++20) for the host runtime, nvcc 12.9 for the sm_90a kernels
(`-gencode arch=compute_90a,code=sm_90a -lineinfo`), one shared object, static cudart so
that the module imports on hosts without a GPU or driver (reference counterpart:
src/Makefile, which has no nvcc step at all).  Objects are cached under build/ by mtime and
compile flags.

    python tools/build_native.py [--force] [--tests] [--jobs N]
"""
from __future__ import annotations

import argparse
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "csrc"
BUILD = ROOT / "build"
PKG = ROOT / "infinistore_b200"

CUDA_HOME = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda"))
NVCC = str(CUDA_HOME / "bin" / "nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]

HOST_SOURCES = [
    "wire/messages.cpp",
    "core/log.cpp",
    "core/mempool.cpp",
    "core/kv_store.cpp",
    "core/trace.cpp",
    "fabric/segment.cpp",
    "fabric/nvls.cpp",
    "fabric/fdpass.cpp",
    "ctrl/server.cpp",
    "ctrl/client.cpp",
    "ctrl/client_data.cpp",
    "ctrl/client_doorbell.cpp",
]
CUDA_SOURCES = [
    "kernels/kv_copy.cu",
    "kernels/kv_pipe.cu",
    "kernels/index_lookup.cu",
    "kernels/kv_read_fused.cu",
    "kernels/kv_fp8.cu",
    "kernels/kv_fp8_records.cu",
    "kernels/kv_fp8_cache.cu",
    "kernels/kv_rope.cu",
    "kernels/kv_fp8_pipe.cu",
    "kernels/kv_doorbell.cu",
    "kernels/kv_bcast_nvls.cu",
]
BINDING = "pybind.cpp"


def _pybind_include() -> str:
    import pybind11

    return pybind11.get_include()


def _ext_suffix() -> str:
    return sysconfig.get_config_var("EXT_SUFFIX") or ".so"


def module_path() -> Path:
    return PKG / f"_infinistore{_ext_suffix()}"


def _newer(src: Path, out: Path, deps: list[Path]) -> bool:
    if not out.exists():
        return True
    t = out.stat().st_mtime
    return any(p.stat().st_mtime > t for p in [src, *deps])


def _headers() -> list[Path]:
    return [p for p in CSRC.rglob("*") if p.suffix in (".h", ".cuh")]


def _run(cmd: list[str]) -> None:
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError(f"build step failed: {cmd[0]} {cmd[-1]}")
    if r.stderr.strip():
        sys.stderr.write(r.stderr)


def build(force: bool = False, jobs: int | None = None, verbose: bool = False) -> Path:
    """Compile everything that is out of date and link the module.  Returns its path."""
    BUILD.mkdir(exist_ok=True)
    hdrs = _headers()
    py_inc = sysconfig.get_paths()["include"]
    common_inc = [f"-I{CSRC}", f"-I{CUDA_HOME / 'include'}"]
    host_flags = ["-std=c++20", "-O2", "-g", "-fPIC", "-Wall", "-Wno-unused-function",
                  "-fvisibility=hidden", "-pthread"]
    nvcc_flags = [*GENCODE, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                  "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]
    # objects built with other flags (e.g. for another architecture) are stale
    stamp = BUILD / "flags.txt"
    flags_id = " ".join([*host_flags, *nvcc_flags])
    if not stamp.exists() or stamp.read_text() != flags_id:
        force = True
    if verbose:
        nvcc_flags += ["-Xptxas", "-v"]

    steps: list[tuple[list[str], Path]] = []
    objs: list[Path] = []
    for rel in HOST_SOURCES:
        src = CSRC / rel
        obj = BUILD / (rel.replace("/", "_") + ".o")
        objs.append(obj)
        if force or _newer(src, obj, hdrs):
            steps.append((["g++", *host_flags, *common_inc, "-c", str(src), "-o", str(obj)], obj))
    for rel in CUDA_SOURCES:
        src = CSRC / rel
        obj = BUILD / (rel.replace("/", "_") + ".o")
        objs.append(obj)
        if force or _newer(src, obj, hdrs):
            steps.append(([NVCC, *nvcc_flags, *common_inc, "-c", str(src), "-o", str(obj)], obj))
    src = CSRC / BINDING
    obj = BUILD / "pybind.o"
    objs.append(obj)
    if force or _newer(src, obj, hdrs):
        steps.append((["g++", *host_flags, *common_inc, f"-I{_pybind_include()}", f"-I{py_inc}",
                       "-c", str(src), "-o", str(obj)], obj))

    if steps:
        with ThreadPoolExecutor(max_workers=jobs or os.cpu_count() or 4) as ex:
            list(ex.map(lambda s: _run(s[0]), steps))

    out = module_path()
    if force or steps or not out.exists():
        tmp = out.with_suffix(".tmp")
        _run(["g++", "-shared", "-o", str(tmp), *map(str, objs),
              f"-L{CUDA_HOME / 'lib64'}", "-lcudart_static", "-lrt", "-ldl", "-lpthread",
              "-Wl,--exclude-libs,ALL"])
        os.replace(tmp, out)
    stamp.write_text(flags_id)
    return out


def build_cpp_tests(force: bool = False, sanitize: bool = False) -> Path:
    """Native unit tests of the core (no Python, no GPU): build/test_core[_san].
    sanitize=True builds with AddressSanitizer + UndefinedBehaviorSanitizer."""
    BUILD.mkdir(exist_ok=True)
    out = BUILD / ("test_core_san" if sanitize else "test_core")
    srcs = [CSRC / "tests" / "test_core.cpp", *(CSRC / s for s in HOST_SOURCES[:4])]
    if force or not out.exists() or any(_newer(s, out, _headers()) for s in srcs):
        flags = ["-std=c++20", "-O1", "-g", "-Wall", "-pthread"]
        if sanitize:
            flags += ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"]
        _run(["g++", *flags, f"-I{CSRC}", f"-I{CUDA_HOME / 'include'}", *map(str, srcs),
              "-o", str(out)])
    return out


def build_loopback_test(force: bool = False, sanitize="address") -> Path:
    """Server + client over loop-back TCP in one native binary (csrc/tests/test_loopback.cpp):
    every host source is compiled with a sanitizer - "address" (ASan + UBSan; True means the
    same), "thread" (TSan: the reactor thread against the client threads) or None - and linked
    against the kernel objects of the regular build (device code is not instrumented; without
    a GPU the CUDA calls fail gracefully and the host-memory pool is used)."""
    build()  # makes sure the kernel objects exist
    if sanitize is True:
        sanitize = "address"
    suffix = {"address": "_san", "thread": "_tsan"}.get(sanitize or "", "")
    out = BUILD / ("test_loopback" + suffix)
    srcs = [CSRC / "tests" / "test_loopback.cpp", *(CSRC / s for s in HOST_SOURCES)]
    kernel_objs = [BUILD / (rel.replace("/", "_") + ".o") for rel in CUDA_SOURCES]
    if force or not out.exists() or any(_newer(s, out, _headers()) for s in srcs):
        flags = ["-std=c++20", "-O1", "-g", "-Wall", "-pthread"]
        if sanitize == "address":
            flags += ["-fsanitize=address,undefined", "-fno-omit-frame-pointer"]
        elif sanitize == "thread":  # std::atomic_thread_fence is not modelled by TSan: say so once
            flags += ["-fsanitize=thread", "-fno-omit-frame-pointer", "-Wno-tsan"]
        _run(["g++", *flags, f"-I{CSRC}", f"-I{CUDA_HOME / 'include'}", *map(str, srcs),
              *map(str, kernel_objs), f"-L{CUDA_HOME / 'lib64'}", "-lcudart_static", "-lrt",
              "-ldl", "-o", str(out)])
    return out


def sass_listing(dst_dir: Path) -> list[Path]:
    """cuobjdump -sass of every kernel object (written to docs/sass/, not committed)."""
    dst_dir.mkdir(parents=True, exist_ok=True)
    written = []
    for rel in CUDA_SOURCES:
        obj = BUILD / (rel.replace("/", "_") + ".o")
        if not obj.exists():
            continue
        r = subprocess.run([str(CUDA_HOME / "bin" / "cuobjdump"), "-sass", str(obj)],
                           capture_output=True, text=True)
        out = dst_dir / (Path(rel).stem + ".sass")
        out.write_text(r.stdout)
        written.append(out)
    return written


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--tests", action="store_true", help="also build the native unit tests")
    ap.add_argument("--jobs", type=int, default=None)
    ap.add_argument("--verbose", action="store_true", help="ptxas -v (registers, spills, smem)")
    ap.add_argument("--sass", action="store_true", help="write SASS listings to docs/sass/")
    ap.add_argument("--clean", action="store_true")
    a = ap.parse_args()
    if a.clean:
        shutil.rmtree(BUILD, ignore_errors=True)
        for p in PKG.glob("_infinistore*.so"):
            p.unlink()
        return
    out = build(force=a.force, jobs=a.jobs, verbose=a.verbose)
    print(out)
    if a.tests:
        print(build_cpp_tests(force=a.force))
    if a.sass:
        for p in sass_listing(ROOT / "docs" / "sass"):
            print(p)


if __name__ == "__main__":
    main()
