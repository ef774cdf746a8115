"""In-tree build of the native libraries (no JIT cache: the .so files travel with the repo).

  avir_b200/libavirb200.so        CUDA kernels + C ABI (include/avirb200.h), sm_90a only
  avir_b200/libavirb200_host.so   the header-only C++ front-ends instantiated behind a C API
                                  (what the Python tests / bench drive)

The oracles (test infrastructure) are built by oracle/Makefile, see build_oracles().
"""
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
INC = os.path.join(ROOT, "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",  # products and sums stay separate IEEE operations (bit-exact contract)
    "-Xcompiler", "-fPIC", "-I" + INC, "-I" + CSRC,
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


class _BuildLock:
    """Serialises builds between processes (parallel test workers import the package at once)."""

    def __enter__(self):
        import fcntl
        self.f = open(os.path.join(PKG, ".build.lock"), "w")
        fcntl.flock(self.f, fcntl.LOCK_EX)
        return self

    def __exit__(self, *a):
        import fcntl
        fcntl.flock(self.f, fcntl.LOCK_UN)
        self.f.close()


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("build failed: " + " ".join(cmd))
    return r.stdout


def _sources(dirs, exts):
    out = []
    for d in dirs:
        for f in sorted(os.listdir(d)):
            if f.endswith(exts):
                out.append(os.path.join(d, f))
    return out


def _obj_stale(obj, src):
    """Per-object staleness from the dependency file nvcc wrote beside it (-MD)."""
    dep = obj + ".d"
    if not os.path.exists(obj) or not os.path.exists(dep):
        return True
    t = os.path.getmtime(obj)
    words = open(dep).read().replace("\\\n", " ").split()
    deps = [w for w in words[1:] if not w.endswith(":")] + [src, os.path.abspath(__file__)]
    for d in deps:
        if d.startswith("/usr/") or d.startswith("/opt/"):
            continue
        if not os.path.exists(d) or os.path.getmtime(d) > t:
            return True
    return False


def build_cuda(force=False, verbose=False):
    with _BuildLock():
        return _build_cuda(force, verbose)


def _build_cuda(force=False, verbose=False):
    """One object per .cu (compiled in parallel, only when one of its own includes changed),
    linked into libavirb200.so."""
    from concurrent.futures import ThreadPoolExecutor
    target = os.path.join(PKG, "libavirb200.so")
    # (source, object, extra flags); stream_chain.cu holds the kernels of ONE pass of ONE streaming
    # chain and is compiled once per chain id (stream_types.h: StreamChainId 1..6) and pass, in parallel
    chains = list(range(1, 8))
    jobs = [(os.path.join(CSRC, n + ".cu"), os.path.join(PKG, n + ".o"), [])
            for n in ("engine", "lancir", "peer_mailbox", "host_call")]
    jobs.append((os.path.join(CSRC, "stream_pass.cu"), os.path.join(PKG, "stream_pass.o"), []))
    jobs += [(os.path.join(CSRC, "stream_chain.cu"), os.path.join(PKG, "stream_chain_%d%s.o" % (k, "hv"[v])),
              ["-DAVS_CHAIN_ID=%d" % k, "-DAVS_CHAIN_PASS=%d" % v]) for k in chains for v in (0, 1)]
    objs = [j[1] for j in jobs]
    todo = [j for j in jobs if force or _obj_stale(j[1], j[0])]

    def compile_one(job):
        cu, obj, extra = job
        tmp = "%s.%d.tmp" % (obj, os.getpid())  # atomic: parallel test workers may build at once
        out = _run([_nvcc()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) +
                   ["-MD", "-MF", tmp + ".d", "-MT", obj, "-c", cu, "-o", tmp])
        os.replace(tmp + ".d", obj + ".d")
        os.replace(tmp, obj)
        return out

    with ThreadPoolExecutor(max_workers=max(2, min(8, os.cpu_count() or 4))) as ex:
        for out in ex.map(compile_one, todo):
            if verbose:
                print(out)
    if todo or not os.path.exists(target):
        tmp = "%s.%d.tmp" % (target, os.getpid())
        _run([_nvcc(), "-shared", "-o", tmp] + objs + ["-lcudart_static", "-ldl", "-lpthread", "-lrt"])
        os.replace(tmp, target)
    return target


def build_host(force=False):
    with _BuildLock():
        return _build_host(force)


def _build_host(force=False):
    target = os.path.join(PKG, "libavirb200_host.so")
    src = os.path.join(CSRC, "host_capi.cpp")
    deps = [src] + _sources([INC], (".h", ".hpp")) + [os.path.join(PKG, "libavirb200.so")]
    if not force and not _newer(target, deps):
        return target
    _run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + INC,
          "-o", target, src, "-L" + PKG, "-lavirb200", "-Wl,-rpath,$ORIGIN", "-pthread"])
    return target


def build_oracles():
    """C port always; the upstream-compiled oracle only where /root/reference exists (oracle/Makefile, and
    oracle/types.mk for CLancIR's double and uint32_t buffers)."""
    _run(["make", "-C", os.path.join(ROOT, "oracle"), "all"])
    _run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "types.mk", "all"])


def build_emul(force=False):
    with _BuildLock():
        return _build_emul(force)


def _build_emul(force=False, name="stream_emul"):
    """TEST INFRASTRUCTURE: host lockstep emulation of the streaming kernel (tests/emul): lib<name>.so
    from <name>.cpp (window_emul.cpp: the windowed passes, on stream_emul.cpp's emulation; config_emul.cpp:
    the generic kernel's shared-memory layout, pass_config.h)."""
    d = os.path.join(ROOT, "tests", "emul")
    target = os.path.join(d, "lib%s.so" % name)
    src = os.path.join(d, name + ".cpp")
    deps = [src, os.path.join(d, "stream_emul.cpp")] + _sources([CSRC, INC], (".cuh", ".h"))
    if not force and not _newer(target, deps):
        return target
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(_nvcc())), "include")
    tmp = "%s.%d.tmp" % (target, os.getpid())  # atomic: parallel test workers may build at once
    _run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + INC, "-I" + CSRC,
          "-I" + cuda_inc, "-o", tmp, src, "-pthread"])
    os.replace(tmp, target)
    return target


def build_window_emul(force=False):
    with _BuildLock():
        return _build_emul(force, "window_emul")


def build_config_emul(force=False):
    with _BuildLock():
        return _build_emul(force, "config_emul")


def build_all(force=False, verbose=False):
    build_cuda(force, verbose)
    build_host(force)
    build_oracles()
    build_emul(force)
    build_window_emul(force)
    build_config_emul(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built")
