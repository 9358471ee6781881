"""Builds viewformer_b200/libvf_b200.so (sm_90a only) with nvcc, in-tree.

    python -m viewformer_b200.build [--force]

nvcc cross-compiles without a GPU; the .so is a build product (git-ignored) and is rebuilt whenever a source or the
public header is newer.  No torch dependency: the library is a plain C-ABI shared object (include/vf_b200.h).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.environ.get("VF_B200_LIB") or os.path.join(HERE, "libvf_b200.so")   # VF_B200_LIB: side-by-side profiling builds
SOURCES = ["vf_misc.cu", "vf_norm.cu", "vf_simt_gemm.cu", "vf_conv_small.cu", "vf_vq.cu", "vf_tc_gemm.cu", "vf_attn_fused.cu", "vf_vq_fused.cu", "vf_eval.cu", "vf_backward.cu", "vf_lpips.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", h) for h in ("vf_b200.h", "vf_b200_pose.h", "vf_b200_lpips.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + [f for f in NVCC_FLAGS if f != "--use_fast_math=false"] + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{out}")
        if verbose and out.strip():
            print(out)
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout)
    if verbose:
        print("built", LIB)
    return LIB


MODEL_LIB = os.path.join(HERE, "libvf_b200_model.so")


def build_model_abi(force=False, verbose=True):
    """libvf_b200_model.so: the model-level C-ABI (include/vf_b200_model.h), a C shim over the embedded interpreter (csrc/vf_model_abi.c).
    Plain gcc; links libpython of the interpreter running this build."""
    import sysconfig
    src = os.path.join(CSRC, "vf_model_abi.c")
    hdr = os.path.join(HERE, "..", "include", "vf_b200_model.h")
    if not force and os.path.exists(MODEL_LIB) and os.path.getmtime(MODEL_LIB) > max(os.path.getmtime(src), os.path.getmtime(hdr)):
        return MODEL_LIB
    gcc = shutil.which("gcc") or shutil.which("cc")
    inc, libdir = sysconfig.get_config_var("INCLUDEPY"), sysconfig.get_config_var("LIBDIR")
    ver = sysconfig.get_config_var("LDVERSION") or sysconfig.get_python_version()
    if not gcc or not inc or not os.path.exists(os.path.join(inc, "Python.h")):
        raise RuntimeError("building libvf_b200_model.so needs gcc and the CPython headers (Python.h)")
    root = os.path.abspath(os.path.join(HERE, ".."))
    cmd = [gcc, "-shared", "-fPIC", "-O2", "-Wall", src, "-I", os.path.join(root, "include"), "-I", inc,
           f'-DVF_PYTHON_DEFAULT="{sys.executable}"', f'-DVF_REPO_ROOT_DEFAULT="{root}"',
           "-L", libdir, f"-lpython{ver}", f"-Wl,-rpath,{libdir}", "-o", MODEL_LIB]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc failed for vf_model_abi.c:\n" + r.stdout)
    if verbose:
        if r.stdout.strip():
            print(r.stdout)
        print("built", MODEL_LIB)
    return MODEL_LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    build_model_abi(force="--force" in sys.argv)
