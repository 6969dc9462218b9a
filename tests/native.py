"""TEST HARNESS ONLY: builds the harness's native code, one recipe per kind, each with its flags written once here.

* restatement: a C restatement (tests/*_ref/*_ref.c, most of which compile the oracle's source in) as a shared library.
* emulator: the product's B2_DEV functions compiled for the CPU (tests/emul/emul.cu, which includes every feature's *_emul.cu, and the
  host BVH build) as one shared library.
* adapter: a C++ adapter program (tests/*_cpp/*.cpp) linked to librmcl_b200.
* nvcc_program: a stand-alone program compiled by nvcc (tests/node_visit).

Outputs go to a per-user directory under the system temporary directory, never into the tree.  Each is named by a hash of its command and
of the content of every file the compiler reads for it, taken from the compiler's own dependency output (-MM), so that an edit to any
source or header it includes gives a new name and a rebuild."""
import ctypes as C
import functools
import hashlib
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
_OUT = os.path.join(tempfile.gettempdir(), f"b2_native_{os.getuid()}")
_GCC = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
_NVCC = os.environ.get("NVCC") or (os.path.join(CUDA, "bin", "nvcc") if os.path.exists(os.path.join(CUDA, "bin", "nvcc")) else "nvcc")
# with -Xcompiler -ffp-contract=off,-mfma on the host: plain float ops are rounded one by one like the device's __fmul_rn / __fadd_rn,
# and fmaf() is a true FMA
_NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false"]


def _build(name, compiler, flags, sources, libs=(), ext=""):
    """compiler flags sources libs -o <_OUT>/<name>_<hash><ext>, unless that file exists; -> its path"""
    h = hashlib.sha1(" ".join([compiler, *flags, *sources, *libs]).encode())
    for src in sources:
        deps = subprocess.run([compiler, *flags, "-MM", src], check=True, capture_output=True, text=True).stdout
        for dep in deps.split(":", 1)[1].replace("\\\n", " ").split():
            with open(dep, "rb") as f:
                h.update(f.read())
    os.makedirs(_OUT, exist_ok=True)
    out = os.path.join(_OUT, f"{name}_{h.hexdigest()[:16]}{ext}")
    if not os.path.exists(out):
        tmp = f"{out}.{os.getpid()}.tmp"
        subprocess.check_call([compiler, *flags, *sources, *libs, "-o", tmp])
        os.replace(tmp, out)
    return out


@functools.cache
def restatement(src):
    """the C restatement tests/<src> as a loaded library; float ops rounded one by one as the oracle's are"""
    path = os.path.join(TESTS, src)
    return C.CDLL(_build(os.path.basename(src)[:-2], _GCC, ["-O2", "-fopenmp", "-ffp-contract=off", "-mavx2", "-mfma", "-fPIC", "-std=gnu11", "-shared"],
                         [path], ["-lm"], ".so"))


@functools.cache
def emulator():
    """the emulator library, loaded once, so that the restype / argtypes its users set are shared"""
    return C.CDLL(_build("emul", _NVCC, _NVCC_FLAGS + ["-Xcompiler", "-fPIC,-fopenmp,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared"],
                         [os.path.join(TESTS, "emul", "emul.cu"), os.path.join(ROOT, "rmcl_b200", "csrc", "bvh_build.cpp")], ["-lgomp"], ".so"))


def adapter(name):
    """the C++ adapter program tests/<name>/<name>.cpp linked to the built librmcl_b200 -> path of the executable"""
    import rmcl_b200
    lib_dir = os.path.dirname(rmcl_b200.lib_path())
    return _build(name, "g++", ["-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(CUDA, "include")],
                  [os.path.join(TESTS, name, name + ".cpp")],
                  ["-L" + lib_dir, "-lrmcl_b200", "-L" + os.path.join(CUDA, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])


def nvcc_program(src):
    """the stand-alone program tests/<src> compiled by nvcc -> path of the executable"""
    return _build(os.path.splitext(os.path.basename(src))[0], _NVCC, _NVCC_FLAGS + ["-Xcompiler", "-ffp-contract=off,-mfma"],
                  [os.path.join(TESTS, src)])
