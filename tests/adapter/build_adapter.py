"""TEST INFRASTRUCTURE: compiles the faiss::Index adapter (faiss_b200/adapter) together with one of its drivers
(tests/adapter/adapter[_<name>]_test.cpp) against the REFERENCE's headers (oracle.ref.REF) and links the reference CPU
library (oracle/_ref) -- the drivers run the reference's own code (faiss::Clustering, faiss::IndexShards, the cloner
pair, IDSelectors, search_and_reconstruct, LocalSearchQuantizer, ResidualQuantizer) over the adapter.  Only possible
where the reference tree is present; the binaries (tests/adapter/_build/adapter[_<name>]_test, git-ignored) travel to
the GPU box with the snapshot."""
import os
import subprocess
import sysconfig

from oracle import ref

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HERE = os.path.join(ROOT, "faiss_b200")
LIB = os.path.join(HERE, "libfaiss_b200.so")

# "" is adapter_test (Clustering, IndexShards, the cloner pair); the others are adapter_<name>_test
DRIVERS = ["", "sel", "recons", "lsq", "rq"]


def driver(name=""):
    return "adapter_%s_test" % name if name else "adapter_test"


def build_adapter(name="", verbose=True):
    """build tests/adapter/_build/adapter[_<name>]_test; returns its path, or None where the reference tree or
    oracle/_ref/libfaiss_ref.so is missing"""
    reflib = ref.LIB_PATH
    if not os.path.isdir(os.path.join(ref.REF, "faiss")) or not os.path.exists(reflib):
        return None
    out = os.path.join(ROOT, "tests", "adapter", "_build", driver(name))
    os.makedirs(os.path.dirname(out), exist_ok=True)
    srcs = [os.path.join(HERE, "adapter", "faiss_b200_adapter.cpp"), os.path.join(ROOT, "tests", "adapter", driver(name) + ".cpp")]
    deps = srcs + [os.path.join(HERE, "adapter", "faiss_b200_adapter.h"), LIB, reflib, os.path.join(ROOT, "include", "faiss_b200_c.h")]
    if os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(f) for f in deps):
        return out
    blasdir = os.path.join(sysconfig.get_paths()["purelib"], "opencv_python_headless.libs")  # OpenBLAS + libgfortran of libfaiss_ref
    cmd = ["/usr/bin/g++", "-std=c++20", "-O2", "-fopenmp", "-w", "-Wl,-rpath-link," + blasdir, "-I" + ref.REF,
           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(HERE, "adapter")] + srcs + [
        "-o", out, reflib, LIB, "-L/usr/local/cuda/lib64", "-lcudart",
        "-Wl,-rpath,$ORIGIN/../../../oracle/_ref:$ORIGIN/../../../faiss_b200:/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("%s failed to build:\n%s\n%s" % (driver(name), r.stdout[-3000:], r.stderr[-3000:]))
    if verbose:
        print("[tests.adapter] built", out, flush=True)
    return out


def build_all(verbose=True):
    """build every driver of DRIVERS, going on past a failure; then raises naming every driver that failed"""
    failed, errors = [], []
    for name in DRIVERS:
        try:
            build_adapter(name, verbose)
        except RuntimeError as e:
            failed.append(driver(name))
            errors.append(str(e))
    if failed:
        raise RuntimeError("adapter drivers %s failed to build:\n%s" % (", ".join(failed), "\n".join(errors)))


if __name__ == "__main__":
    build_all()
