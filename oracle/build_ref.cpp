// TEST INFRASTRUCTURE — not part of the product.
//
// Compiles the UNMODIFIED reference kernels from where they lie under
// /root/reference into cubins under oracle/_ref/, replicating the reference's
// own run-time compilation pipeline:
//   NVRTC per module with the reference's flag set  (include/CudaModularProgram.h:84-98)
//   nvJitLink -dlto -arch=sm_<device>               (include/CudaModularProgram.h:214-239)
// The reference does this at run time on the device it finds; the build needs no
// GPU, so the link target is given on the command line (sm_90 for an H100).
// No reference source is copied into this repository: the sources are read in
// place and only the compiled cubins are written (oracle/_ref/ is git-ignored).
//
// usage: build_ref <reference_root> <out_dir> <sm_arch, e.g. 90>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>
#include <nvrtc.h>
#include <nvJitLink.h>

static std::string readFile(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) { std::cerr << "cannot read " << path << "\n"; exit(2); }
    std::stringstream ss; ss << f.rdbuf(); return ss.str();
}

struct Ltoir { std::vector<char> data; };

static Ltoir compileModule(const std::string& path, const std::string& dir, const std::string& cudaInc) {
    std::string src = readFile(path);
    nvrtcProgram prog;
    nvrtcCreateProgram(&prog, src.c_str(), path.c_str(), 0, nullptr, nullptr);
    std::string incDir = "-I " + dir;
    std::string incCuda = "-I " + cudaInc;
    // flag set of CudaModularProgram.h:84-98, verbatim (arch stays compute_89: LTO-IR is retargeted at link)
    std::vector<const char*> opts = {
        "--gpu-architecture=compute_89",
        "--use_fast_math",
        "--extra-device-vectorization",
        "-lineinfo",
        incCuda.c_str(),
        incDir.c_str(),
        "-I ./",
        "--relocatable-device-code=true",
        "-default-device",
        "-dlto",
        "--std=c++20",
        "--disable-warnings",
    };
    nvrtcResult res = nvrtcCompileProgram(prog, (int)opts.size(), opts.data());
    if (res != NVRTC_SUCCESS) {
        size_t n; nvrtcGetProgramLogSize(prog, &n); std::string log(n, 0); nvrtcGetProgramLog(prog, log.data());
        std::cerr << "NVRTC failed for " << path << "\n" << log << "\n"; exit(3);
    }
    Ltoir out; size_t n = 0; nvrtcGetLTOIRSize(prog, &n); out.data.resize(n); nvrtcGetLTOIR(prog, out.data.data());
    nvrtcDestroyProgram(&prog);
    return out;
}

static void linkProgram(const std::vector<Ltoir>& mods, const std::string& arch, const std::string& outPath) {
    std::string strArch = "-arch=sm_" + arch;
    const char* lopts[] = {"-dlto", strArch.c_str()};
    nvJitLinkHandle h;
    if (nvJitLinkCreate(&h, 2, lopts) != NVJITLINK_SUCCESS) { std::cerr << "nvJitLinkCreate failed\n"; exit(4); }
    for (auto& m : mods)
        if (nvJitLinkAddData(h, NVJITLINK_INPUT_LTOIR, (void*)m.data.data(), m.data.size(), "module label") != NVJITLINK_SUCCESS) {
            std::cerr << "nvJitLinkAddData failed\n"; exit(4);
        }
    if (nvJitLinkComplete(h) != NVJITLINK_SUCCESS) {
        size_t n = 0; nvJitLinkGetErrorLogSize(h, &n); std::string log(n, 0); nvJitLinkGetErrorLog(h, log.data());
        std::cerr << "nvJitLinkComplete failed\n" << log << "\n"; exit(4);
    }
    size_t n = 0; nvJitLinkGetLinkedCubinSize(h, &n); std::vector<char> cubin(n); nvJitLinkGetLinkedCubin(h, cubin.data());
    nvJitLinkDestroy(&h);
    std::ofstream f(outPath, std::ios::binary); f.write(cubin.data(), cubin.size());
    std::cout << "wrote " << outPath << " (" << n << " bytes)\n";
}

int main(int argc, char** argv) {
    if (argc < 4) { std::cerr << "usage: build_ref <reference_root> <out_dir> <sm_arch>\n"; return 1; }
    std::string root = argv[1], out = argv[2], arch = argv[3];
    std::string dir = root + "/modules/progressive_octree";
    const char* cp = getenv("CUDA_PATH");
    std::string cudaInc = std::string(cp ? cp : "/usr/local/cuda") + "/include";
    // the three programs of main_progressive_octree.cpp:603-626
    struct Prog { const char* out; std::vector<const char*> mods; };
    std::vector<Prog> progs = {
        {"ref_construct.cubin", {"progressive_octree_voxels.cu", "utils.cu"}},
        {"ref_reset.cubin",     {"reset.cu", "utils.cu"}},
        {"ref_render.cubin",    {"render.cu", "utils.cu"}},
    };
    for (auto& p : progs) {
        std::vector<Ltoir> mods;
        for (auto m : p.mods) mods.push_back(compileModule(dir + "/" + m, dir, cudaInc));
        linkProgram(mods, arch, out + "/" + p.out);
    }
    return 0;
}
