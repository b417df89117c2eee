"""Build recipes for the engine (nvcc, sm_90a only: H100) and for the test-side artefacts.

Everything is built IN-TREE, so the package and the tests run from the source tree:
  lightning_b200/libcln_sigverify.so   the product (CUDA kernels + C ABI; its plain-C parts by gcc) [nvcc]
  tests/host_emul/libemul.so           kernel headers compiled for the host, tests only [g++]
  oracle/libsecp_port.so               the plain-C restatement oracle                 [gcc]
  oracle/_ref/libsecp_ref.so           the unmodified reference, from the Core Lightning tree at $CLN_SRC or /root/reference [gcc]
  lightning_b200/cln_sigverifyd, cln_verify_gossip_store   the verifier subdaemon and the gossip_store audit tool [gcc]
  oracle/_ref/libcln_ref.so, libcln_bolt12.so, libcln_gossmap.so   CLN's own plumbing, BOLT12 Merkle code and
                                        gossip_store loader (common/gossmap.c) from the same tree [gcc]
  oracle/_ref/libcln_funding.so         CLN's funding script (bitcoin/script.c bitcoin_redeem_2of2) from the same tree [gcc]
  oracle/_ref/libcln_bolt11.so          CLN's BOLT11 decoder (common/bolt11.c bolt11_decode) from the same tree [gcc]
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "lightning_b200", "csrc")
LIB = os.path.join(ROOT, "lightning_b200", "libcln_sigverify.so")
EMUL = os.path.join(ROOT, "tests", "host_emul", "libemul.so")
DAEMON = os.path.join(ROOT, "lightning_b200", "cln_sigverifyd")
STORE_TOOL = os.path.join(ROOT, "lightning_b200", "cln_verify_gossip_store")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    # curve-side kernel: inlined field arithmetic + CTA-wide re-convergence barriers (see fe.cuh and common.cuh)
    "-DSV_FE_INLINE", "-DSV_MAIN_SYNC",
]
# gcc flags of the plain-C parts: the drop-in (linked into the library) and the verifier subdaemon
DROPIN_CFLAGS = ["-O2", "-fPIC", "-Wall", "-Wextra", "-std=c11"]
DAEMON_CFLAGS = ["-O2", "-Wall", "-Wextra", "-std=c11", "-pthread"]
# g++ line of the host build of the kernel headers (tests only; tests/invalid_curve.py builds altered copies with it)
HOST_EMUL_CXX = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wall", "-Wno-unused-function"]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _sources(d, exts):
    out = []
    for base, _, files in os.walk(d):
        out += [os.path.join(base, f) for f in files if f.endswith(exts)]
    return out


def build_engine(force=False, verbose=False):
    srcs = _sources(CSRC, (".cu", ".cuh", ".c", ".h")) + [os.path.join(ROOT, "include", "cln_sigverify.h"),
                                                   os.path.join(ROOT, "include", "cln_dropin.h")]
    # the flags are part of what the library is: a change of flags must rebuild, and so must a stale daemon
    stamp = os.path.join(os.path.dirname(LIB), ".build_flags")
    flags_now = " ".join(NVCC_FLAGS)
    same_flags = os.path.exists(stamp) and open(stamp).read() == flags_now
    if not force and same_flags and _newer(LIB, srcs) and _newer(DAEMON, srcs) and _newer(STORE_TOOL, srcs):
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    # host side of the drop-in is plain C (as the reference's bitcoin/signature.c), compiled by gcc
    dropin_o = os.path.join(CSRC, "cln_dropin.o")
    r = subprocess.run(["gcc"] + DROPIN_CFLAGS + ["-c", os.path.join(CSRC, "cln_dropin.c"), "-o", dropin_o], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc (cln_dropin.c) failed:\n" + r.stdout + r.stderr)
    # pruning a gossip_store file in place (sv_prune_gossip_store_fd): plain C over the engine's prune entry points
    store_fd_o = os.path.join(CSRC, "gossip_store_fd.o")
    r = subprocess.run(["gcc"] + DROPIN_CFLAGS + ["-c", os.path.join(CSRC, "gossip_store_fd.c"), "-o", store_fd_o],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc (gossip_store_fd.c) failed:\n" + r.stdout + r.stderr)
    # salvaging a gossip_store file in place (sv_salvage_gossip_store_fd): plain C over the salvage and the repair
    salvage_fd_o = os.path.join(CSRC, "gossip_salvage_fd.o")
    r = subprocess.run(["gcc"] + DROPIN_CFLAGS + ["-c", os.path.join(CSRC, "gossip_salvage_fd.c"), "-o", salvage_fd_o],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc (gossip_salvage_fd.c) failed:\n" + r.stdout + r.stderr)
    # the batch-verification kernels are a translation unit of their own, compiled with the field multiplier as real
    # functions (see batch.cu); everything else inlines it
    batch_flags = [f for f in NVCC_FLAGS if f not in ("-shared", "-DSV_FE_INLINE", "-DSV_MAIN_SYNC")] + ["-DSV_NO_SYNC_INLINE", "-c"]
    batch_o = os.path.join(CSRC, "batch.o")
    r = subprocess.run([nvcc] + batch_flags + (["-Xptxas", "-v"] if verbose else []) + ["-o", batch_o, os.path.join(CSRC, "batch.cu")],
                       capture_output=True, text=True)
    if verbose:
        sys.stderr.write(r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc (batch.cu) failed:\n" + r.stdout + r.stderr)
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [
        "-o", LIB, os.path.join(CSRC, "engine.cu"), batch_o, dropin_o, store_fd_o, salvage_fd_o]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose:
        sys.stderr.write(r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    # verifier subdaemon (row N4): plain C, links the engine
    r = subprocess.run(["gcc"] + DAEMON_CFLAGS + [os.path.join(CSRC, "sigverifyd.c"), "-o", DAEMON,
                        "-L" + os.path.dirname(LIB), "-lcln_sigverify", "-Wl,-rpath,$ORIGIN"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc (sigverifyd.c) failed:\n" + r.stdout + r.stderr)
    # gossip_store audit tool: plain C, links the engine
    r = subprocess.run(["gcc"] + DAEMON_CFLAGS + [os.path.join(CSRC, "cln_verify_gossip_store.c"), "-o", STORE_TOOL,
                        "-L" + os.path.dirname(LIB), "-lcln_sigverify", "-Wl,-rpath,$ORIGIN"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("gcc (cln_verify_gossip_store.c) failed:\n" + r.stdout + r.stderr)
    open(stamp, "w").write(flags_now)
    return LIB


def build_host_emul(force=False):
    src = [os.path.join(ROOT, "tests", "host_emul", f) for f in ("emul.cpp", "bolt12_emul.cpp", "gossip_store_emul.cpp",
                                                             "gossip_funding_emul.cpp", "fee_grind_emul.cpp",
                                                             "gossip_salvage_emul.cpp", "bolt11_emul.cpp")]
    srcs = _sources(CSRC, (".cuh",)) + src
    if not force and _newer(EMUL, srcs):
        return EMUL
    cmd = HOST_EMUL_CXX + ["-o", EMUL] + src
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ (host_emul) failed:\n" + r.stdout + r.stderr)
    return EMUL


def build_oracle():
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "all"], capture_output=True, text=True,
                       stdin=subprocess.DEVNULL, timeout=900)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + r.stdout + r.stderr)
    # the reference's BOLT12 Merkle code, linked against the library above
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "bolt12.mk", "all"], capture_output=True, text=True,
                       stdin=subprocess.DEVNULL, timeout=900)
    if r.returncode != 0:
        raise RuntimeError("oracle build (bolt12.mk) failed:\n" + r.stdout + r.stderr)
    # the reference's gossip_store loader (common/gossmap.c), with the configurator's config.h of the `cln` target
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "gossmap.mk", "all"], capture_output=True, text=True,
                       stdin=subprocess.DEVNULL, timeout=900)
    if r.returncode != 0:
        raise RuntimeError("oracle build (gossmap.mk) failed:\n" + r.stdout + r.stderr)
    # the same loader as gossipd loads its store at start-up (strict), linked with the objects above
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "gossmap_strict.mk", "all"], capture_output=True,
                       text=True, stdin=subprocess.DEVNULL, timeout=900)
    if r.returncode != 0:
        raise RuntimeError("oracle build (gossmap_strict.mk) failed:\n" + r.stdout + r.stderr)
    # the reference's funding script (bitcoin/script.c, bitcoin/pubkey.c), linked with the plumbing objects of the `cln` target
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "funding.mk", "all"], capture_output=True,
                       text=True, stdin=subprocess.DEVNULL, timeout=900)
    if r.returncode != 0:
        raise RuntimeError("oracle build (funding.mk) failed:\n" + r.stdout + r.stderr)
    # the reference's BOLT11 decoder (common/bolt11.c), linked against the library of the `cln` target
    r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "bolt11.mk", "all"], capture_output=True,
                       text=True, stdin=subprocess.DEVNULL, timeout=900)
    if r.returncode != 0:
        raise RuntimeError("oracle build (bolt11.mk) failed:\n" + r.stdout + r.stderr)


def build_all(force=False, verbose=False):
    build_engine(force=force, verbose=verbose)
    build_host_emul(force=force)
    build_oracle()


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print("built:", LIB)
