"""Build recipe for the native parts (no torch involved).

  simlod_b200/csrc/{construct,render,reset,util,las,partition,gen,export,import,query,pick,nearest,ray,radius,las_write,heightmap}.cu  --nvcc sm_90a-->  build/*.cubin
  build/*.cubin --bin2c--> build/*_cubin.c  (embedded images)
  simlod_b200/csrc/host.cpp + images --g++--> simlod_b200/libsimlod_b200.so   (the C ABI, include/simlod_b200.h)
  build/*.cubin are also copied to simlod_b200/cubin/ : the drop-in artefacts for the reference's
  own host (INTEGRATION.md).

The library is kept in-tree (git-ignored) so that the package imports from the source tree.
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "simlod_b200", "csrc")
BUILD = os.path.join(ROOT, "build")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA, "bin", "nvcc")
BIN2C = os.path.join(CUDA, "bin", "bin2c")
LIB = os.path.join(ROOT, "simlod_b200", "libsimlod_b200.so")
CUBIN_DIR = os.path.join(ROOT, "simlod_b200", "cubin")
PROGRAMS = ["construct", "render", "reset", "util", "las", "partition", "gen", "export", "import", "query", "pick", "nearest", "ray", "radius",
            "las_write", "heightmap"]
# gen.cu restates numpy generators in IEEE double arithmetic: no mul+add contraction
EXTRA_FLAGS = {"gen": ["--fmad=false"]}
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
REF_ARCH = "90"


def _run(cmd, **kw):
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if res.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + res.stdout + "\n")
        raise RuntimeError("build step failed: " + " ".join(cmd[:3]))
    return res.stdout


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _digest(paths, extra=""):
    """Content hash of the inputs of a build step: freshness must not depend on mtimes or on the intermediate
    build/ directory, neither of which survives a copy of the tree to another machine (the built artefacts and the stamp do)."""
    import hashlib
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        h.update(os.path.relpath(p, ROOT).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stamp_matches(stamp, digest, artefacts):
    try:
        return all(os.path.exists(a) for a in artefacts) and open(stamp).read().strip() == digest
    except OSError:
        return False


def build_native(force=False, verbose=False):
    headers = [os.path.join(ROOT, "include", "simlod_abi.h"), os.path.join(ROOT, "include", "simlod_b200.h"),
               os.path.join(CSRC, "fpmath.cuh"), os.path.join(CSRC, "lodcut.cuh"), os.path.join(CSRC, "loader_pool.h"),
               os.path.join(CSRC, "construct_layout.cuh"), os.path.join(CSRC, "export_common.cuh"), os.path.join(CSRC, "region.cuh"),
               os.path.join(CSRC, "search_common.cuh"),
               os.path.join(CSRC, "kernel_args.h"), os.path.join(CSRC, "render_layout.cuh"), os.path.join(CSRC, "render_frame.inc"),
               os.path.join(CSRC, "splat.cuh")]
    sources = [os.path.join(CSRC, name + ".cu") for name in PROGRAMS] + [os.path.join(CSRC, "host.cpp")]
    digest = _digest(sources + headers, " ".join(ARCH) + " -O3 -lineinfo " + repr(sorted(EXTRA_FLAGS.items())))
    stamp = os.path.join(CUBIN_DIR, "BUILD_STAMP")
    artefacts = [LIB] + [os.path.join(CUBIN_DIR, "simlod_%s.cubin" % name) for name in PROGRAMS]
    if not force and _stamp_matches(stamp, digest, artefacts):
        return LIB
    os.makedirs(BUILD, exist_ok=True)
    os.makedirs(CUBIN_DIR, exist_ok=True)
    images = []
    for name in PROGRAMS:
        src = os.path.join(CSRC, name + ".cu")
        cubin = os.path.join(BUILD, name + ".cubin")
        if force or not _newer(cubin, [src] + headers):
            out = _run([NVCC] + ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + EXTRA_FLAGS.get(name, []) + ["-cubin", "-o", cubin, src])
            if verbose:
                print(out)
        shutil.copyfile(cubin, os.path.join(CUBIN_DIR, "simlod_%s.cubin" % name))
        cfile = os.path.join(BUILD, name + "_cubin.c")
        if force or not _newer(cfile, [cubin]):
            text = _run([BIN2C, "--const", "--padd", "0", "--name", "simlod_cubin_" + name, cubin])
            # bin2c emits a static-less definition guarded for C++; keep it plain C with external linkage
            with open(cfile, "w") as f:
                f.write(text)
        images.append(cfile)
    host = os.path.join(CSRC, "host.cpp")
    if force or not _newer(LIB, [host] + images + headers):
        objs = []
        for c in images:
            o = c[:-2] + ".o"
            _run(["gcc", "-c", "-O1", "-fPIC", c, "-o", o])
            objs.append(o)
        _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I" + os.path.join(CUDA, "include"), host] + objs +
             ["-o", LIB, "-ldl"])
    with open(stamp, "w") as f:
        f.write(digest + "\n")
    return LIB


def build_oracle(force=False):
    """Compile the CPU restatement (oracle/liboracle.so) and, when the reference tree is present,
    the reference's own kernels into oracle/_ref/*.cubin. Checker infrastructure only."""
    odir = os.path.join(ROOT, "oracle")
    lib = os.path.join(odir, "liboracle.so")
    srcs = [os.path.join(odir, f) for f in ("oracle.cpp",)]
    odigest = _digest(srcs + [os.path.join(ROOT, "include", "simlod_abi.h")], "-O2 -ffp-contract=off")
    ostamp = lib + ".stamp"
    if force or not _stamp_matches(ostamp, odigest, [lib]):
        _run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include")] + srcs + ["-o", lib])
        with open(ostamp, "w") as f:
            f.write(odigest + "\n")
    ref_root = os.environ.get("SIMLOD_REFERENCE", "/root/reference")
    refdir = os.path.join(odir, "_ref")
    if os.path.isdir(os.path.join(ref_root, "modules", "progressive_octree")):
        os.makedirs(refdir, exist_ok=True)
        tool = os.path.join(refdir, "build_ref")
        tool_src = os.path.join(odir, "build_ref.cpp")
        if force or not _newer(tool, [tool_src]):
            _run(["g++", "-O1", "-std=c++17", tool_src, "-I" + os.path.join(CUDA, "include"), "-L" + os.path.join(CUDA, "lib64"),
                  "-lnvrtc", "-lnvJitLink", "-Wl,-rpath," + os.path.join(CUDA, "lib64"), "-o", tool])
        # the reference's CPU LAS loader: LasLoader.cpp compiles from its own single source file
        las = os.path.join(refdir, "libref_las.so")
        shim = os.path.join(odir, "ref_las_shim.cpp")
        if force or not _newer(las, [shim]):
            po = os.path.join(ref_root, "modules", "progressive_octree")
            _run(["g++", "-O2", "-std=c++20", "-fPIC", "-shared", "-w", "-I" + po, "-I" + os.path.join(ref_root, "include"),
                  "-I" + os.path.join(ref_root, "libs", "fmt", "include"), os.path.join(po, "LasLoader.cpp"), shim, "-o", las, "-pthread"])
        # ... and its .simlod loader (SimlodLoader.cpp needs <cstdint> force-included, SURVEY.md §8c)
        sml = os.path.join(refdir, "libref_simlod.so")
        shim2 = os.path.join(odir, "ref_simlod_shim.cpp")
        if force or not _newer(sml, [shim2]):
            po = os.path.join(ref_root, "modules", "progressive_octree")
            _run(["g++", "-O2", "-std=c++20", "-fPIC", "-shared", "-w", "-include", "cstdint", "-I" + po, "-I" + os.path.join(ref_root, "include"),
                  "-I" + os.path.join(ref_root, "libs", "fmt", "include"), os.path.join(po, "SimlodLoader.cpp"), shim2, "-o", sml, "-pthread"])
        # the reference links for the device it runs on (sm_90 on an H100)
        outs = [os.path.join(refdir, n) for n in ("ref_construct.cubin", "ref_render.cubin", "ref_reset.cubin")]
        rstamp = os.path.join(refdir, "ref_cubins.stamp")
        if force or not _stamp_matches(rstamp, REF_ARCH, outs):
            _run([tool, ref_root, refdir, REF_ARCH], cwd=odir)
            with open(rstamp, "w") as f:
                f.write(REF_ARCH + "\n")
    return lib


def build_test_harness(force=False):
    """tests/native/dropin_harness: the reference host's launch sequence over the shipped cubins (driver API only, linked
    against the toolkit's stub libcuda so that it builds on a machine without a driver). Test infrastructure."""
    src = os.path.join(ROOT, "tests", "native", "dropin_harness.cpp")
    out = os.path.join(ROOT, "tests", "native", "dropin_harness")
    if not os.path.exists(src):
        return None
    digest = _digest([src, os.path.join(ROOT, "include", "simlod_abi.h")], "-O1")
    stamp = out + ".stamp"
    if force or not _stamp_matches(stamp, digest, [out]):
        _run(["g++", "-O1", "-std=c++17", "-I" + os.path.join(CUDA, "include"), src, "-o", out,
              "-L" + os.path.join(CUDA, "lib64", "stubs"), "-lcuda"])
        with open(stamp, "w") as f:
            f.write(digest + "\n")
    return out


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose=True))
    if os.path.exists(os.path.join(ROOT, "oracle", "oracle.cpp")):
        print(build_oracle(force="--force" in sys.argv))
    print(build_test_harness(force="--force" in sys.argv))
