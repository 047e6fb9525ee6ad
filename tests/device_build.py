"""The build of the test kernels under tests/devicelogic/: each compiles with nvcc for sm_90a against include/ alone, so
that it sees the public headers and nothing of the engine's sources.  Importing this module starts no CUDA context."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
NVCC = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-I", INCLUDE]


def compile_so(name, outdir, extra=()):
    """nvcc tests/devicelogic/<name>.cu into outdir/<name>.so; returns (path, nvcc's output)"""
    so = os.path.join(outdir, name + ".so")
    src = os.path.join(HERE, "devicelogic", name + ".cu")
    p = subprocess.run(NVCC + ["-shared", "-Xcompiler", "-fPIC", *extra, "-o", so, src], capture_output=True, text=True,
                       check=True)
    return so, p.stdout + p.stderr


def load(build):
    """the shared library build(dir) writes into a temporary directory and returns the path of, loaded; the directory
    is removed (the loaded library outlives its file)"""
    tmp = tempfile.mkdtemp(prefix="devicelogic_")
    try:
        return C.CDLL(build(tmp))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def load_kernel(name):
    """tests/devicelogic/<name>.cu, compiled into a temporary directory and loaded"""
    return load(lambda d: compile_so(name, d)[0])
