"""In-tree build of the sm_90a extension ``distributed_training_guide_b200/_C.so``.

    python -m distributed_training_guide_b200.build [--force] [--verbose]

Every ``csrc/*.cu`` is compiled by nvcc for ``-gencode arch=compute_90a,code=sm_90a
-lineinfo`` (cross-compiles without a GPU), ``csrc/*.cpp`` by g++ against the torch headers,
and everything is linked into one shared object next to this file so that it travels with
the repository snapshot to the GPU box (a JIT cache under ~/.cache would not).  The kernels
do not include torch headers, so a .cu rebuild takes seconds.
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import hashlib
import os
import shlex
import subprocess
import sys
import sysconfig
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OBJ = HERE / "build" / "obj"
TARGET = HERE / "_C.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "--expt-extended-lambda", "-Xcompiler", "-fPIC",
    "-Xptxas", "-v", "-DNDEBUG",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
             "-D_GLIBCXX_USE_CXX11_ABI=1", "-Wno-deprecated-declarations"]


def cuda_home() -> Path:
    for k in ("CUDA_HOME", "CUDA_PATH"):
        if os.environ.get(k):
            return Path(os.environ[k])
    return Path("/usr/local/cuda")


def _run(cmd, verbose, log_path=None):
    if verbose:
        print(" ".join(shlex.quote(str(c)) for c in cmd), flush=True)
    r = subprocess.run([str(c) for c in cmd], capture_output=True, text=True)
    if log_path is not None:
        Path(log_path).write_text(r.stdout + r.stderr)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f"build step failed: {' '.join(map(str, cmd))}")
    return r.stdout + r.stderr


def _stamp(src: Path, flags) -> str:
    h = hashlib.sha1()
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))):
        h.update(hdr.read_bytes())
    h.update(" ".join(flags).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    import torch
    from torch.utils import cpp_extension as ce

    OBJ.mkdir(parents=True, exist_ok=True)
    cuda = cuda_home()
    nvcc = cuda / "bin" / "nvcc"
    torch_inc = [f"-I{p}" for p in ce.include_paths()]
    py_inc = f"-I{sysconfig.get_paths()['include']}"
    cuda_inc = f"-I{cuda / 'include'}"
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cxx_flags = [f.replace("ABI=1", f"ABI={abi}") for f in CXX_FLAGS]

    jobs = []
    for src in sorted(CSRC.glob("*.cu")):
        obj = OBJ / (src.stem + ".cu.o")
        flags = NVCC_FLAGS + [cuda_inc, f"-I{CSRC}"]
        jobs.append((src, obj, [nvcc, *flags, "-c", src, "-o", obj], flags))
    for src in sorted(CSRC.glob("*.cpp")):
        obj = OBJ / (src.stem + ".cpp.o")
        flags = cxx_flags + torch_inc + [py_inc, cuda_inc, f"-I{CSRC}"]
        jobs.append((src, obj, ["g++", *flags, "-c", src, "-o", obj], flags))

    def compile_one(job):
        src, obj, cmd, flags = job
        stamp_file = obj.with_suffix(obj.suffix + ".stamp")
        stamp = _stamp(src, [str(f) for f in flags])
        if not force and obj.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
            return False
        _run(cmd, verbose, log_path=obj.with_suffix(obj.suffix + ".log"))
        stamp_file.write_text(stamp)
        return True

    with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 4)) as ex:
        rebuilt = list(ex.map(compile_one, jobs))

    if any(rebuilt) or not TARGET.exists() or force:
        torch_lib = Path(torch.__file__).parent / "lib"
        link = ["g++", "-shared", "-o", TARGET, *[j[1] for j in jobs],
                f"-L{torch_lib}", f"-Wl,-rpath,{torch_lib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda",
                "-ltorch", "-ltorch_python",
                f"-L{cuda / 'lib64'}", f"-Wl,-rpath,{cuda / 'lib64'}", "-lcudart", "-ldl", "-lpthread"]
        _run(link, verbose)
    return TARGET


def ptxas_report() -> str:
    """registers / spills / shared memory per kernel, from the saved nvcc -Xptxas -v logs."""
    out = []
    for log in sorted(OBJ.glob("*.cu.o.log")):
        out.append(f"== {log.name}")
        out.append(log.read_text())
    return "\n".join(out)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--ptxas", action="store_true", help="print the ptxas -v report after building")
    a = ap.parse_args()
    t = build(a.force, a.verbose)
    print(f"built {t}")
    if a.ptxas:
        print(ptxas_report())
