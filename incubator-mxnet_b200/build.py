"""Build the in-tree native library ``incubator-mxnet_b200/libmxkv_b200.so`` for sm_90a (H100).

nvcc cross-compiles without a GPU; the library and its objects are build products (git-ignored).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libmxkv_b200.so")
SOURCES = ["kernels.cu", "tree_kernels.cu", "rsp_kernels.cu", "norm_kernels.cu", "kvstore_norm.cc", "runtime.cc", "vmm_arena.cc", "topology.cc", "ndarray.cc", "kvstore.cc", "kvstore_rsp.cc", "c_api.cc"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall", "--threads", "4"]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "include", "mxkv_b200.h"))
    deps.append(os.path.abspath(__file__))
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(HERE, "build", src.rsplit(".", 1)[0] + ".o")
        cmd = [NVCC] + FLAGS + ["-x", "cu", "-c", path, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed on %s:\n%s\n" % (src, out.decode()))
        elif verbose and out:
            print(out.decode())
    if failed:
        raise RuntimeError("native build failed")
    cmd = [NVCC, "-shared", "-o", OUT] + objs + GENCODE
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
