"""Build libanovos_b200.so in-tree with nvcc for sm_90a (H100; no GPU needed: nvcc cross-compiles).

    python -m anovos_b200.build            # incremental
    python -m anovos_b200.build --force
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libanovos_b200.so")
SOURCES = ["capi.cu", "scan_host.cu", "scan_mom.cu", "scan_hist.cu", "scan_fused.cu", "scan_assign.cu", "drift.cu", "synth.cu", "select.cu", "hll.cu", "sort.cu", "sample.cu", "gk_host.cu", "rows.cu", "impute.cu", "scale.cu", "encode.cu", "transform.cu", "invalid.cu"]
# transform.cu restates fdlibm, which specifies no fused multiply-add: its products and sums are rounded one by one
EXTRA_FLAGS = {"transform.cu": ["-fmad=false"]}
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17"] + GENCODE + ["-lineinfo",
              "--expt-relaxed-constexpr", "--expt-extended-lambda", "-Xcompiler", "-fPIC,-O3",
              "-Xptxas", "-v"]


def _nvcc():
    for p in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if p and (os.path.isabs(p) and os.path.exists(p) or not os.path.isabs(p)):
            return p
    return "nvcc"


def source_hash():
    """sha1 over every kernel source + the public header, in name order."""
    import hashlib
    h = hashlib.sha1()
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h")))
    files.append(os.path.join(os.path.dirname(HERE), "include", "anovos_b200.h"))
    for f in files:
        h.update(os.path.basename(f).encode())
        h.update(open(f, "rb").read())
    return h.hexdigest()


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_variant(tag, defines):
    """Experimental build with extra -D flags -> anovos_b200/build/variants/libanovos_b200_<tag>.so"""
    vdir = os.path.join(HERE, "build", "variants", tag)
    os.makedirs(vdir, exist_ok=True)
    objs, procs = [], []
    for s in SOURCES:
        obj = os.path.join(vdir, s.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [_nvcc()] + [f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")] + EXTRA_FLAGS.get(s, []) + \
              ["-D" + d for d in defines] + \
              ["-c", os.path.join(CSRC, s), "-o", obj]
        procs.append(subprocess.Popen(cmd))
    if any(p.wait() != 0 for p in procs):
        raise RuntimeError("nvcc failed for variant " + tag)
    lib = os.path.join(HERE, "build", "variants", "libanovos_b200_%s.so" % tag)
    subprocess.check_call([_nvcc(), "-shared", "-o", lib] + objs + GENCODE)
    return lib


def build(force=False, verbose=False):
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "anovos_b200.h"))
    objs, procs = [], []
    digest = source_hash()
    stamp = os.path.join(objdir, "source_hash.txt")
    old_digest = open(stamp).read().strip() if os.path.exists(stamp) else ""
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        objs.append(obj)
        extra = []
        stale = force or _stale(obj, [src] + headers)
        if s == "capi.cu":      # carries the hash of ALL sources: recompiled (cheap) whenever any of them changed
            extra = ['-DANV_SOURCE_HASH="%s"' % digest]
            stale = stale or digest != old_digest
        if stale:
            cmd = [_nvcc()] + NVCC_FLAGS + EXTRA_FLAGS.get(s, []) + extra + ["-c", src, "-o", obj]
            log = open(obj + ".log", "w")
            procs.append((s, subprocess.Popen(cmd, stdout=log, stderr=subprocess.STDOUT), obj + ".log"))
    failed = False
    for s, p, logf in procs:
        rc = p.wait()
        if rc != 0 or verbose:
            sys.stderr.write(open(logf).read())
        if rc != 0:
            failed = True
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(LIB, objs):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + GENCODE
        subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
