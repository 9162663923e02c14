"""In-tree build of ``unicore_b200._C`` (one extension, sm_90a only).

Two entry points share the same source list and flags:
* ``build_inplace()`` - used by ``__graft_entry__.build()``: compiles every ``.cu`` with
  ``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` (no PyTorch headers needed there, a few
  seconds each, in parallel), the binding ``.cpp`` files with the host compiler against the PyTorch
  headers, and links ``unicore_b200/_C<abi-suffix>.so`` next to the Python sources so that the
  artefact travels with the repository snapshot.  Objects are cached by source mtime.
* ``cuda_extension()`` / ``build_ext_class()`` - the same thing expressed as a setuptools
  ``CUDAExtension`` for ``python setup.py build_ext --inplace``.
"""
import concurrent.futures
import glob
import os
import shutil
import subprocess
import sys
import sysconfig

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CSRC = os.path.join(ROOT, "csrc")
OBJ_DIR = os.path.join(ROOT, "build", "obj")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17", "--use_fast_math",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-Wno-deprecated-declarations"]


def sources():
    cu = sorted(glob.glob(os.path.join(CSRC, "**", "*.cu"), recursive=True))
    cpp = sorted(glob.glob(os.path.join(CSRC, "**", "*.cpp"), recursive=True))
    return cu, cpp


def so_path():
    suffix = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return os.path.join(ROOT, "unicore_b200", "_C" + suffix)


def _headers_mtime():
    hs = glob.glob(os.path.join(CSRC, "**", "*.h"), recursive=True) + glob.glob(
        os.path.join(CSRC, "**", "*.cuh"), recursive=True
    )
    return max([os.path.getmtime(h) for h in hs] + [0.0])


def _obj_for(src):
    rel = os.path.relpath(src, CSRC).replace(os.sep, "__")
    return os.path.join(OBJ_DIR, rel + ".o")


def _stale(src, obj, hdr_mtime):
    return (not os.path.exists(obj)) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_mtime)


def _run(cmd):
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise RuntimeError("command failed: {}\n{}".format(" ".join(cmd), proc.stdout))
    return proc.stdout


def _torch_paths():
    import torch
    from torch.utils import cpp_extension

    includes = cpp_extension.include_paths(device_type="cuda")
    libdirs = cpp_extension.library_paths(device_type="cuda")
    abi = int(getattr(torch._C, "_GLIBCXX_USE_CXX11_ABI", True))
    return includes, libdirs, abi


def build_inplace(verbose=False, force=False):
    """Compile + link ``unicore_b200/_C*.so``. Returns the path of the shared object."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cxx = os.environ.get("CXX", "g++")
    os.makedirs(OBJ_DIR, exist_ok=True)
    # objects built with other flags (another architecture, another compiler) are never reused
    stamp = os.path.join(OBJ_DIR, "flags.txt")
    flags = "\n".join([nvcc, cxx] + NVCC_FLAGS + CXX_FLAGS)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    cu, cpp = sources()
    hdr_mtime = _headers_mtime()
    includes, libdirs, abi = _torch_paths()
    py_inc = sysconfig.get_paths()["include"]
    jobs = []
    for src in cu:
        obj = _obj_for(src)
        if force or _stale(src, obj, hdr_mtime):
            jobs.append([nvcc] + NVCC_FLAGS + ["-I", CSRC, "-c", src, "-o", obj])
    inc_flags = []
    for inc in includes + [py_inc, CSRC]:
        inc_flags += ["-I", inc]
    for src in cpp:
        obj = _obj_for(src)
        if force or _stale(src, obj, hdr_mtime):
            jobs.append(
                [cxx] + CXX_FLAGS + inc_flags
                + ["-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
                   "-D_GLIBCXX_USE_CXX11_ABI={}".format(abi), "-c", src, "-o", obj]
            )
    if jobs:
        workers = min(len(jobs), max(1, (os.cpu_count() or 4)))
        with concurrent.futures.ThreadPoolExecutor(max_workers=workers) as pool:
            for out in pool.map(_run, jobs):
                if verbose and out.strip():
                    print(out)
    target = so_path()
    objs = [_obj_for(s) for s in cu + cpp]
    # relink whenever the library is missing or older than an object (e.g. an earlier link failed)
    stale_so = not os.path.exists(target) or any(os.path.getmtime(o) > os.path.getmtime(target) for o in objs)
    if force or jobs or stale_so:
        link = [cxx, "-shared", "-o", target] + objs
        for d in libdirs:
            link += ["-L", d, "-Wl,-rpath," + d]
        cuda_lib = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "lib64")
        link += ["-L", cuda_lib, "-Wl,-rpath," + cuda_lib]
        link += ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart", "-lcuda"]
        # The shared libstdc++ that torch uses, named explicitly: where the compiler's own libstdc++.so link is missing,
        # g++'s implicit -lstdc++ falls back to libstdc++.a, and a second, static copy of the stream and locale code
        # in the extension crashes the process as soon as an error message formats a number.
        link += ["-l:libstdc++.so.6"]
        _run(link)
    # only a complete build (compiled and linked with these flags) is recorded
    with open(stamp, "w") as f:
        f.write(flags)
    return target


def cuda_extension():
    from torch.utils.cpp_extension import CUDAExtension

    cu, cpp = sources()
    rel = [os.path.relpath(s, ROOT) for s in cu + cpp]
    return CUDAExtension(
        name="unicore_b200._C",
        sources=rel,
        include_dirs=[CSRC],
        extra_compile_args={"cxx": CXX_FLAGS, "nvcc": NVCC_FLAGS},
        libraries=["cuda"],
        extra_link_args=["-l:libstdc++.so.6"],  # (see build_inplace)
    )


def build_ext_class():
    from torch.utils.cpp_extension import BuildExtension

    return BuildExtension.with_options(use_ninja=True)


if __name__ == "__main__":
    print(build_inplace(verbose="-v" in sys.argv, force="-f" in sys.argv))
