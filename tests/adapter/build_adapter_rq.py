"""TEST INFRASTRUCTURE: compiles the adapter's B200ResidualQuantizer and B200ProgressiveDimIndexFactory with their
driver (tests/adapter/adapter_rq_test.cpp) against the REFERENCE's headers and CPU library (oracle/_ref), as
tests/adapter/build_adapter.py does for adapter_test.cpp.  The binary (tests/adapter/_build/adapter_rq_test, git-ignored) travels to the GPU box with the
snapshot."""
import os
import subprocess
import sysconfig

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HERE = os.path.join(ROOT, "faiss_b200")
LIB = os.path.join(HERE, "libfaiss_b200.so")
OUT = os.path.join(ROOT, "tests", "adapter", "_build", "adapter_rq_test")


def build_adapter_rq(verbose=True):
    ref = "/root/reference"
    reflib = os.path.join(ROOT, "oracle", "_ref", "libfaiss_ref.so")
    if not os.path.isdir(os.path.join(ref, "faiss")) or not os.path.exists(reflib):
        return None
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    srcs = [os.path.join(HERE, "adapter", "faiss_b200_adapter.cpp"), os.path.join(ROOT, "tests", "adapter", "adapter_rq_test.cpp")]
    deps = srcs + [os.path.join(HERE, "adapter", "faiss_b200_adapter.h"), LIB, reflib, os.path.join(ROOT, "include", "faiss_b200_c.h")]
    if os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(f) for f in deps):
        return OUT
    blasdir = os.path.join(sysconfig.get_paths()["purelib"], "opencv_python_headless.libs")  # OpenBLAS of libfaiss_ref
    cmd = ["/usr/bin/g++", "-std=c++20", "-O2", "-fopenmp", "-w", "-Wl,-rpath-link," + blasdir, "-I" + ref,
           "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(HERE, "adapter")] + srcs + [
        "-o", OUT, reflib, LIB, "-L/usr/local/cuda/lib64", "-lcudart",
        "-Wl,-rpath,$ORIGIN/../../../oracle/_ref:$ORIGIN/../../../faiss_b200:/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("adapter RQ driver build failed:\n%s\n%s" % (r.stdout[-3000:], r.stderr[-3000:]))
    if verbose:
        print("[tests.adapter] built", OUT, flush=True)
    return OUT


if __name__ == "__main__":
    print(build_adapter_rq())
