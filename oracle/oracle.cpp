// oracle.cpp — TEST INFRASTRUCTURE. CPU restatement of the reference's octree builder and
// rasteriser, used only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg as the
// checker. Nothing in simlod_b200/ includes, links or calls this file.
//
// Pinning (see oracle/README.md and DESIGN.md §6): the reference ships no tests, golden vectors or
// fixtures (SURVEY.md §4), so this restatement is pinned against the reference's OWN kernels:
//   * on the GPU, tests/test_parity_gpu.py compares with oracle/_ref/*.cubin (the unmodified reference
//     sources compiled by oracle/build_ref.cpp) on the same inputs and compares canonical forms;
//   * tests/golden/*.npz holds canonical digests produced by those reference kernels on an H100
//     (generator: tests/golden/make_golden.py); the CPU-only suite checks this file against them.
//
// The builder follows the reference phase by phase, serially:
//   addBatch          progressive_octree_voxels.cu:700-802   (phase order)
//   expand            :385-415      doCounting :124-306      doSplitting :308-383
//   voxelSampling     :417-483      sampleVoxel :50-121
//   allocatePointChunks :485-538    allocateVoxelChunks :641-672
//   insertPoints      :540-639      insertVoxels :674-698
//   reset             reset.cu:20-86
// Arithmetic follows the reference's SASS on sm_90 (see simlod_b200/csrc/fpmath.cuh): plain
// mul/add/fma are IEEE round-to-nearest without flush; a/b is a*MUFU.RCP(b) with the product
// flushed; float->uint saturates and flushes. MUFU.RCP cannot be reproduced on a CPU: it is exact
// for powers of two (all CPU-only test cubes are 2^k); for other cube sizes the caller passes the
// device's value (simlod_device_rcp). In the rasteriser 1/w is taken as the correctly rounded
// reciprocal, so CPU pixel coordinates can differ from the GPU's in rare boundary cases; render
// parity of record is GPU-vs-reference-kernel, bit-exact (tests/test_parity_gpu.py).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <unordered_map>
#include <unordered_set>
#include <vector>
#include "simlod_abi.h"

namespace {

typedef SimlodPoint Point;

constexpr uint32_t MAXP = SIMLOD_MAX_POINTS_PER_NODE;
constexpr uint32_t PPC = SIMLOD_POINTS_PER_CHUNK;
constexpr int MAX_DEPTH = SIMLOD_MAX_DEPTH;

// ---- float primitives --------------------------------------------------------------------------
inline float ftz(float v) { return std::fabs(v) < 1.17549435e-38f ? std::copysign(0.0f, v) : v; }
inline float mul_ftz(float a, float b) { return ftz(a * b); }
inline uint32_t f2u(float v) {               // F2I.FTZ.U32.TRUNC: saturating, NaN -> 0
    v = ftz(v);
    if (!(v == v)) return 0;
    if (v <= 0.0f) return 0;
    if (v >= 4294967296.0f) return 0xffffffffu;
    return (uint32_t)v;
}
inline int32_t f2i(float v) {
    v = ftz(v);
    if (!(v == v)) return 0;
    if (v >= 2147483648.0f) return 0x7fffffff;
    if (v <= -2147483648.0f) return (int32_t)0x80000000;
    return (int32_t)v;
}
inline int32_t d2i(double v) {
    if (!(v == v)) return 0;
    if (v >= 2147483648.0) return 0x7fffffff;
    if (v <= -2147483648.0) return (int32_t)0x80000000;
    return (int32_t)v;
}
inline float ex2neg(uint32_t level) { return std::ldexp(1.0f, -(int)level); }   // MUFU.EX2(-level): exact

struct Coords { uint32_t X, Y, Z, pX, pY, pZ; };

struct Quantizer {
    float minx, miny, minz, size, rcp;
    Coords operator()(const Point& p) const {      // voxels.cu:148-155
        float dx = p.x - minx, dy = p.y - miny, dz = p.z - minz;
        Coords q;
        q.X = f2u(mul_ftz(dx * 1048576.0f, rcp));
        q.Y = f2u(mul_ftz(dy * 1048576.0f, rcp));
        q.Z = f2u(mul_ftz(dz * 1048576.0f, rcp));
        q.pX = f2u(mul_ftz(dx * 268435456.0f, rcp));
        q.pY = f2u(mul_ftz(dy * 268435456.0f, rcp));
        q.pZ = f2u(mul_ftz(dz * 268435456.0f, rcp));
        return q;
    }
};
inline uint32_t childIndexAt(const Coords& q, int level) {      // voxels.cu:171-179
    int sh = MAX_DEPTH - level - 1;
    return (((q.X >> sh) & 1u) << 2) | (((q.Y >> sh) & 1u) << 1) | ((q.Z >> sh) & 1u);
}
inline uint32_t cellAt(const Coords& q, uint32_t level) {       // voxels.cu:78-88
    uint32_t sh = (MAX_DEPTH + 1) - level;
    return ((q.pX >> sh) & 127u) | (((q.pY >> sh) & 127u) << 7) | (((q.pZ >> sh) & 127u) << 14);
}

// ---- the oracle's octree ----------------------------------------------------------------------
struct ONode {
    int32_t children[8];
    uint32_t counter = 0, numPoints = 0, level = 0, X = 0, Y = 0, Z = 0, countIteration = 0;
    uint8_t name[24];
    bool hasGrid = false;
    std::vector<uint32_t> grid;           // 65536 words when hasGrid
    uint32_t numPointChunks = 0;          // length of the points chunk list
    uint32_t numVoxelChunks = 0;
    std::vector<Point> points;            // stored points, slot order
    std::vector<Point> voxels;            // stored voxels, slot order
    std::vector<uint32_t> voxelCells;     // cell of voxels[i]
    std::vector<uint32_t> voxelBatch;     // batch index that created voxels[i]
    uint32_t numVoxels = 0, numVoxelsStored = 0;
    ONode() { for (auto& c : children) c = -1; memset(name, 0, sizeof(name)); }
    bool isLeaf() const { for (int c : children) if (c >= 0) return false; return true; }
};

struct OStats {
    uint32_t numNodes, numInner, numLeaves, numNonemptyLeaves, numPoints, numVoxels, numChunksPoints, numChunksVoxels;
    uint32_t batchletIndex, droppedSpilledPoints;
    uint64_t numPointsProcessed, numAllocatedChunks, chunkPoolSize, allocatedBytes_persistent;
};

struct Backlog { Point voxel; int32_t target; uint32_t cell; };

struct Oracle {
    Quantizer q;
    std::vector<ONode> nodes;
    uint64_t heapOffset = 16;
    uint64_t numAllocatedChunks = 0, chunkPoolSize = 0;
    uint32_t batchletIndex = 0;
    uint64_t numPointsProcessed = 0;
    uint32_t dropped = 0;
    // (node << 21 | cell) -> colours of the points that could have created that voxel, per creation
    std::vector<std::pair<uint64_t, uint32_t>> colorCandidates;
    bool candidatesSorted = false;

    uint64_t heapAlloc(uint64_t size) { uint64_t o = heapOffset; heapOffset += 16ull * ((size + 16ull) / 16ull); return o; }   // utils.h.cu:185-197

    void reset() {                                   // reset.cu:40-83
        nodes.clear(); nodes.emplace_back();
        ONode& root = nodes[0];
        root.name[0] = 'r';
        heapOffset = 16;
        root.hasGrid = true; root.grid.assign(SIMLOD_GRID_WORDS, 0); heapAlloc(sizeof(SimlodOccupancyGrid));
        numAllocatedChunks = chunkPoolSize = 0; batchletIndex = 0; numPointsProcessed = 0; dropped = 0;
        colorCandidates.clear(); candidatesSorted = false;
    }

    int32_t findLeaf(const Coords& c) const {        // voxels.cu:157-189
        int32_t cur = 0;
        for (int level = 0; level < MAX_DEPTH; level++) {
            int32_t ch = nodes[cur].children[childIndexAt(c, level)];
            if (ch < 0) break;
            cur = ch;
        }
        return cur;
    }

    // voxels.cu:124-306. Returns true when no leaf spilled.
    bool doCounting(const Point* pts, uint32_t n, std::vector<Point>& spilled, std::vector<int32_t>& spilling, uint32_t countIteration) {
        spilling.clear();
        auto countPoint = [&](const Point& p) {
            int32_t leaf = findLeaf(q(p));
            ONode& L = nodes[leaf];
            if (L.countIteration < countIteration) {
                uint32_t old = L.counter++;
                if (old <= MAXP && old + 1 > MAXP) spilling.push_back(leaf);     // :211-217, group size 1
            }
        };
        for (uint32_t i = 0; i < n; i++) countPoint(pts[i]);
        size_t numSpilledBefore = spilled.size();
        for (size_t i = 0; i < numSpilledBefore; i++) countPoint(spilled[i]);
        for (int32_t s : spilling) {                                             // :253-289
            ONode& node = nodes[s];
            for (uint32_t i = 0; i < node.numPoints; i++) spilled.push_back(node.points[i]);
        }
        for (auto& nd : nodes) nd.countIteration = countIteration;              // :298-300
        return spilling.empty();
    }

    void doSplitting(const std::vector<int32_t>& spilling) {                     // voxels.cu:308-383
        for (int32_t s : spilling) {
            int32_t childOffset = (int32_t)nodes.size();
            nodes.resize(nodes.size() + 8);
            ONode& sp = nodes[s];
            for (int i = 0; i < 8; i++) {
                ONode& child = nodes[childOffset + i];
                child.level = sp.level + 1;
                child.X = 2 * sp.X + ((i >> 2) & 1);
                child.Y = 2 * sp.Y + ((i >> 1) & 1);
                child.Z = 2 * sp.Z + (i & 1);
                memcpy(child.name, sp.name, 20);
                if (child.level < 24) child.name[child.level] = (uint8_t)(i + '0');
                sp.children[i] = childOffset + i;
            }
            numAllocatedChunks -= sp.numPointChunks;                             // chunks go back to the pool (:345-357)
            sp.numPointChunks = 0; sp.numPoints = 0; sp.points.clear();
            if (!sp.hasGrid) { sp.hasGrid = true; heapAlloc(sizeof(SimlodOccupancyGrid)); }
            sp.grid.assign(SIMLOD_GRID_WORDS, 0);                                // :370-382 clears the grid of EVERY split node (root's too)
        }
    }

    void expand(const Point* pts, uint32_t n, std::vector<Point>& spilled) {     // voxels.cu:385-415
        std::vector<int32_t> spilling;
        for (int i = 0; i < 20; i++) {
            bool finished = doCounting(pts, n, spilled, spilling, batchletIndex + 1);
            if (finished) break;
            doSplitting(spilling);
        }
    }

    void sampleVoxel(int32_t n, const Coords& c, const Point& p, std::vector<Backlog>& backlog, std::unordered_set<uint64_t>& created) {   // voxels.cu:50-121
        ONode& node = nodes[n];
        if (!node.hasGrid) return;
        uint32_t cell = cellAt(c, node.level);
        uint32_t& word = node.grid[cell >> 5];
        uint32_t bit = 1u << (cell & 31u);
        if (word & bit) return;
        word |= bit;
        node.numVoxels++;
        float nodeSize = mul_ftz(ex2neg(node.level), q.size);
        float vx = std::fmaf(nodeSize, (float)node.X, q.minx) + mul_ftz(nodeSize * ((float)(cell & 127u) + 0.5f), 0.0078125f);
        float vy = std::fmaf(nodeSize, (float)node.Y, q.miny) + mul_ftz(nodeSize * ((float)((cell >> 7) & 127u) + 0.5f), 0.0078125f);
        float vz = std::fmaf(nodeSize, (float)node.Z, q.minz) + mul_ftz(nodeSize * ((float)((cell >> 14) & 127u) + 0.5f), 0.0078125f);
        backlog.push_back(Backlog{Point{vx, vy, vz, p.color}, n, cell});
        created.insert(((uint64_t)n << 21) | cell);
    }

    template <typename F>
    void forEachPathNode(const Coords& c, F&& f) {                               // voxels.cu:449-469
        int32_t cur = 0;
        for (int level = 0; level < MAX_DEPTH; level++) {
            f(cur);
            int32_t ch = nodes[cur].children[childIndexAt(c, level)];
            if (ch < 0) break;
            cur = ch;
        }
    }

    void addBatch(const Point* pts, uint32_t n) {                                // voxels.cu:700-802
        std::vector<Point> spilled;
        std::vector<Backlog> backlog;
        expand(pts, n, spilled);

        // voxelSampling (:417-483): batch points, then spilled points
        std::unordered_set<uint64_t> created;
        auto sampleAll = [&](const Point& p) { Coords c = q(p); forEachPathNode(c, [&](int32_t nd) { sampleVoxel(nd, c, p, backlog, created); }); };
        for (uint32_t i = 0; i < n; i++) sampleAll(pts[i]);
        for (const Point& p : spilled) sampleAll(p);
        // colour candidates: on the GPU the creating point of a cell is whichever of these raced first
        auto collect = [&](const Point& p) {
            Coords c = q(p);
            forEachPathNode(c, [&](int32_t nd) {
                if (!nodes[nd].hasGrid) return;
                uint64_t key = ((uint64_t)nd << 21) | cellAt(c, nodes[nd].level);
                if (created.count(key)) colorCandidates.emplace_back(key, p.color);
            });
        };
        for (uint32_t i = 0; i < n; i++) collect(pts[i]);
        for (const Point& p : spilled) collect(p);
        candidatesSorted = false;

        // allocatePointChunks (:485-538)
        for (auto& node : nodes) {
            if (!node.isLeaf() || !(node.numPoints < node.counter)) continue;
            uint32_t required = (node.counter + PPC - 1) / PPC, existing = (node.numPoints + PPC - 1) / PPC;
            for (uint32_t i = existing; i < required; i++) {
                uint64_t chunkIndex = numAllocatedChunks++;
                if (chunkIndex >= chunkPoolSize) heapAlloc(sizeof(SimlodChunk));   // else: taken from the pool
                node.numPointChunks++;
            }
        }
        chunkPoolSize = std::max(chunkPoolSize, numAllocatedChunks);

        // allocateVoxelChunks (:641-672)
        for (auto& node : nodes) {
            uint32_t required = (node.numVoxels + PPC - 1) / PPC;
            while (node.numVoxelChunks < required) { heapAlloc(sizeof(SimlodChunk)); node.numVoxelChunks++; }
        }

        // insertPoints (:540-639)
        auto insertPoint = [&](const Point& p) { ONode& L = nodes[findLeaf(q(p))]; L.points.push_back(p); L.numPoints++; };
        for (uint32_t i = 0; i < n; i++) insertPoint(pts[i]);
        for (size_t i = 0; i < spilled.size(); i++) {
            if (i > 3000000) { dropped++; continue; }                            // :628-631 (sic)
            insertPoint(spilled[i]);
        }
        // insertVoxels (:674-698)
        for (const Backlog& b : backlog) {
            ONode& t = nodes[b.target];
            t.voxels.push_back(b.voxel); t.voxelCells.push_back(b.cell); t.voxelBatch.push_back(batchletIndex);
            t.numVoxelsStored++;
        }
        batchletIndex++;                                                          // :925-928
        numPointsProcessed += n;
    }

    OStats stats() const {                                                        // voxels.cu:958-1009
        OStats s{};
        s.numNodes = (uint32_t)nodes.size();
        for (const auto& node : nodes) {
            if (node.isLeaf()) {
                s.numLeaves++; s.numPoints += node.numPoints; s.numChunksPoints += (node.numPoints + PPC - 1) / PPC;
                if (node.numPoints > 0) s.numNonemptyLeaves++;
            } else {
                s.numInner++; s.numVoxels += node.numVoxels; s.numChunksVoxels += (node.numVoxels + PPC - 1) / PPC;
            }
        }
        s.batchletIndex = batchletIndex; s.droppedSpilledPoints = dropped; s.numPointsProcessed = numPointsProcessed;
        s.numAllocatedChunks = numAllocatedChunks; s.chunkPoolSize = chunkPoolSize; s.allocatedBytes_persistent = heapOffset;
        return s;
    }
};

// ---- canonical form (shared by the oracle tree and a downloaded device image) ------------------
struct CNode {
    int32_t children[8];
    uint32_t level, X, Y, Z, counter, numPoints, numVoxels, numVoxelsStored;
    uint8_t name[20];
    uint32_t chunksPoints, chunksVoxels;
    std::vector<Point> points, voxels;
    uint8_t visible = 0, isLarge = 0;
    bool isLeaf() const { for (int c : children) if (c >= 0) return false; return true; }
};

struct CanonRecord {
    uint32_t level, X, Y, Z;
    uint8_t name[20];
    uint32_t counter, numPoints, numVoxels, numVoxelsStored;
    uint32_t isLeaf, chunksPoints, chunksVoxels, nodeIndex;
    uint64_t hashPoints;      // sorted multiset of 16-byte points
    uint64_t hashVoxelPos;    // sorted multiset of 12-byte voxel positions
};

struct Canon {
    std::vector<CNode> nodes;
    std::vector<uint32_t> order;      // node indices sorted by (level, X, Y, Z)
    int error = 0;
};

inline bool pointLess(const Point& a, const Point& b) { return memcmp(&a, &b, 16) < 0; }
inline bool posLess(const Point& a, const Point& b) { return memcmp(&a, &b, 12) < 0; }

uint64_t hashBytes(uint64_t h, const void* data, size_t n) {      // FNV-1a 64
    const uint8_t* p = (const uint8_t*)data;
    for (size_t i = 0; i < n; i++) { h ^= p[i]; h *= 0x100000001b3ull; }
    return h;
}

void finalizeCanon(Canon& c) {
    c.order.resize(c.nodes.size());
    for (uint32_t i = 0; i < c.nodes.size(); i++) c.order[i] = i;
    std::sort(c.order.begin(), c.order.end(), [&](uint32_t a, uint32_t b) {
        const CNode &A = c.nodes[a], &B = c.nodes[b];
        if (A.level != B.level) return A.level < B.level;
        if (A.X != B.X) return A.X < B.X;
        if (A.Y != B.Y) return A.Y < B.Y;
        return A.Z < B.Z;
    });
}

Canon* canonFromOracle(const Oracle& o) {
    Canon* c = new Canon();
    c->nodes.resize(o.nodes.size());
    for (size_t i = 0; i < o.nodes.size(); i++) {
        const ONode& s = o.nodes[i];
        CNode& d = c->nodes[i];
        memcpy(d.children, s.children, sizeof(d.children));
        d.level = s.level; d.X = s.X; d.Y = s.Y; d.Z = s.Z; d.counter = s.counter; d.numPoints = s.numPoints;
        d.numVoxels = s.numVoxels; d.numVoxelsStored = s.numVoxelsStored;
        memcpy(d.name, s.name, 20);
        d.chunksPoints = s.numPointChunks; d.chunksVoxels = s.numVoxelChunks;
        d.points = s.points; d.voxels = s.voxels;
    }
    finalizeCanon(*c);
    return c;
}

// walk a raw device image: nodes[] bytes + persistent heap bytes, pointers are device addresses
Canon* canonFromImage(const uint8_t* nodesBytes, uint64_t numNodes, const uint8_t* heap, uint64_t heapBytes, uint64_t nodesAddr, uint64_t heapAddr) {
    Canon* c = new Canon();
    c->nodes.resize(numNodes);
    auto readChunks = [&](uint64_t first, uint32_t count, std::vector<Point>& out, uint32_t& numChunks) {
        numChunks = 0;
        uint64_t addr = first;
        uint32_t left = count;
        while (addr != 0) {
            if (addr < heapAddr || addr + sizeof(SimlodChunk) > heapAddr + heapBytes) { c->error = 2; return; }
            const SimlodChunk* ch = (const SimlodChunk*)(heap + (addr - heapAddr));
            uint32_t take = std::min(left, PPC);
            out.insert(out.end(), ch->points, ch->points + take);
            left -= take;
            numChunks++;
            if (numChunks > 10000000u) { c->error = 3; return; }
            addr = (uint64_t)ch->next;
        }
        if (left != 0) c->error = 4;        // list shorter than the element count
    };
    for (uint64_t i = 0; i < numNodes; i++) {
        const SimlodNode* s = (const SimlodNode*)(nodesBytes + i * sizeof(SimlodNode));
        CNode& d = c->nodes[i];
        for (int k = 0; k < 8; k++) {
            uint64_t a = (uint64_t)s->children[k];
            if (a == 0) d.children[k] = -1;
            else if (a < nodesAddr || (a - nodesAddr) % sizeof(SimlodNode) != 0 || (a - nodesAddr) / sizeof(SimlodNode) >= numNodes) { c->error = 1; d.children[k] = -1; }
            else d.children[k] = (int32_t)((a - nodesAddr) / sizeof(SimlodNode));
        }
        d.level = s->level; d.X = s->X; d.Y = s->Y; d.Z = s->Z; d.counter = s->counter; d.numPoints = s->numPoints;
        d.numVoxels = s->numVoxels; d.numVoxelsStored = s->numVoxelsStored;
        memcpy(d.name, s->name, 20);
        d.visible = s->visible; d.isLarge = s->isLarge;
        readChunks((uint64_t)s->points, s->numPoints, d.points, d.chunksPoints);
        readChunks((uint64_t)s->voxelChunks, s->numVoxelsStored, d.voxels, d.chunksVoxels);
    }
    finalizeCanon(*c);
    return c;
}

// ---- CPU rasteriser (render.cu:61-104,161-210,690-934,1126-1131) --------------------------------
struct Row { float x, y, z, w; };
inline float rcpf(float v) { return ftz(1.0f / v); }     // stands in for MUFU.RCP (see header)
inline float rowDot(const SimlodFloat4& r, float x, float y, float z) { return r.w + std::fmaf(z, r.z, std::fmaf(x, r.x, y * r.y)); }
inline float dot3(float ax, float ay, float az, float bx, float by, float bz) { return std::fmaf(az, bz, std::fmaf(ax, bx, ay * by)); }

bool planeRejects(float px, float py, float pz, float pw, const float* mn, const float* mx) {   // math.cuh:55-64,184-198
    float len = std::sqrt(dot3(px, py, pz, px, py, pz));
    float inv = rcpf(len);
    float nx = mul_ftz(px, inv), ny = mul_ftz(py, inv), nz = mul_ftz(pz, inv), cst = mul_ftz(pw, inv);
    float vx = nx > 0.0f ? mx[0] : mn[0], vy = ny > 0.0f ? mx[1] : mn[1], vz = nz > 0.0f ? mx[2] : mn[2];
    return (dot3(nx, ny, nz, vx, vy, vz) + cst) < 0.0f;
}

struct RenderStats { uint32_t numVisibleNodes, numVisibleInner, numVisibleLeaves, numVisiblePoints, numVisibleVoxels; };

void renderCanon(Canon& c, const SimlodUniforms& u, uint64_t* fb, RenderStats* rs) {
    const int width = f2i(u.width), height = f2i(u.height);
    for (int64_t i = 0; i < (int64_t)width * height; i++) fb[i] = (0x7f800000ull << 32) | 0x00332211ull;
    float cubeSize = std::max(std::max(u.boxMax[0] - u.boxMin[0], u.boxMax[1] - u.boxMin[1]), u.boxMax[2] - u.boxMin[2]);
    const SimlodFloat4* T = u.transform_updateBound.rows;
    // pass 1: flags (render.cu:762-901)
    for (CNode& node : c.nodes) {
        float nodeSize = mul_ftz(cubeSize, ex2neg(node.level));
        float f[3] = {(float)node.X, (float)node.Y, (float)node.Z};
        float mn[3], mx[3];
        for (int a = 0; a < 3; a++) { mn[a] = std::fmaf(nodeSize, f[a], u.boxMin[a]); mx[a] = std::fmaf(nodeSize, f[a] + 1.0f, u.boxMin[a]); }
        float sminx = 0, smaxx = 0, sminy = 0, smaxy = 0;
        for (int corner = 0; corner < 8; corner++) {
            float x = (corner & 4) ? mx[0] : mn[0], y = (corner & 2) ? mx[1] : mn[1], z = (corner & 1) ? mx[2] : mn[2];
            float rw = rcpf(rowDot(T[3], x, y, z));
            float sx = u.width * std::fmaf(mul_ftz(rowDot(T[0], x, y, z), rw), 0.5f, 0.5f);
            float sy = u.height * std::fmaf(mul_ftz(rowDot(T[1], x, y, z), rw), 0.5f, 0.5f);
            if (corner == 0) { sminx = smaxx = sx; sminy = smaxy = sy; }
            else { sminx = std::fmin(sminx, sx); smaxx = std::fmax(smaxx, sx); sminy = std::fmin(sminy, sy); smaxy = std::fmax(smaxy, sy); }
        }
        float dx = smaxx - sminx, dy = smaxy - sminy;
        bool inFrustum = true;
        for (int p = 0; p < 6 && inFrustum; p++) {
            const SimlodFloat4& a = T[3];
            const SimlodFloat4& b = T[(p == 0 || p == 1) ? 0 : ((p == 2 || p == 3) ? 1 : 2)];
            float sgn = (p == 0 || p == 3 || p == 4) ? -1.0f : 1.0f;
            if (planeRejects(a.x + sgn * b.x, a.y + sgn * b.y, a.z + sgn * b.z, a.w + sgn * b.w, mn, mx)) inFrustum = false;
        }
        bool hasSamples = node.numPoints > 0 || node.numVoxels > 0;
        double limit = 2.0 * (double)u.minNodeSize;
        node.visible = inFrustum && hasSamples;
        node.isLarge = (double)dx > limit || (double)dy > limit;
    }
    // pass 2 + draw (render.cu:906-933, 61-104)
    RenderStats st{};
    const SimlodFloat4* M = u.transform.rows;
    auto drawSamples = [&](const std::vector<Point>& pts, uint32_t count) {
        for (uint32_t i = 0; i < count && i < pts.size(); i++) {
            const Point& p = pts[i];
            float w = rowDot(M[3], p.x, p.y, p.z);
            float rw = rcpf(w);
            float ndcx = mul_ftz(rowDot(M[0], p.x, p.y, p.z), rw), ndcy = mul_ftz(rowDot(M[1], p.x, p.y, p.z), rw);
            int x = d2i(std::fma((double)ndcx, 0.5, 0.5) * (double)u.width);
            int y = d2i(std::fma((double)ndcy, 0.5, 0.5) * (double)u.height);
            if (!(x > 1 && (double)x < (double)u.width - 2.0 && y > 1 && (double)y < (double)u.height - 2.0)) continue;
            uint32_t ud; memcpy(&ud, &w, 4);
            uint64_t enc = ((uint64_t)ud << 32) | p.color;
            for (int ox = 0; ox < u.pointSize; ox++)
            for (int oy = 0; oy < u.pointSize; oy++) {
                uint32_t px = (uint32_t)std::max(0, std::min(x + ox, width)), py = (uint32_t)std::max(0, std::min(y + oy, height));
                uint64_t id = px + (uint64_t)width * py;
                if (id < (uint64_t)width * height && enc < fb[id]) fb[id] = enc;
            }
        }
    };
    auto makeVisible = [&](const CNode& node) {
        st.numVisibleNodes++;
        if (node.numPoints > 0) { st.numVisibleLeaves++; st.numVisiblePoints += node.numPoints; }
        else if (node.numVoxels > 0) { st.numVisibleInner++; st.numVisibleVoxels += node.numVoxels; }
        if (u.showPoints) { drawSamples(node.points, node.numPoints); drawSamples(node.voxels, node.numVoxels); }
    };
    for (const CNode& node : c.nodes) {
        if (node.isLarge && !node.isLeaf()) {
            for (int i = 0; i < 8; i++) {
                if (node.children[i] < 0) continue;
                const CNode& child = c.nodes[node.children[i]];
                if (child.isLarge || !child.visible) continue;
                makeVisible(child);
            }
        } else if (node.isLarge && node.isLeaf() && node.visible) {
            makeVisible(node);
        }
    }
    if (rs) *rs = st;
}

}  // namespace

// ---- C interface for ctypes -----------------------------------------------------------------------
extern "C" {

void* oracle_create(const float* boxMin, const float* boxMax, float rcpSize) {
    Oracle* o = new Oracle();
    float size = std::max(std::max(boxMax[0] - boxMin[0], boxMax[1] - boxMin[1]), boxMax[2] - boxMin[2]);   // voxels.cu:860-863
    o->q = Quantizer{boxMin[0], boxMin[1], boxMin[2], size, rcpSize != 0.0f ? rcpSize : 1.0f / size};
    o->reset();
    return o;
}
void oracle_destroy(void* h) { delete (Oracle*)h; }
void oracle_reset(void* h) { ((Oracle*)h)->reset(); }
int oracle_add_batch(void* h, const SimlodPoint* pts, uint32_t n) { ((Oracle*)h)->addBatch(pts, n); return 0; }
void oracle_get_stats(void* h, OStats* out) { *out = ((Oracle*)h)->stats(); }

void* canon_from_oracle(void* h) { return canonFromOracle(*(Oracle*)h); }
void* canon_from_image(const uint8_t* nodes, uint64_t numNodes, const uint8_t* heap, uint64_t heapBytes, uint64_t nodesAddr, uint64_t heapAddr) {
    return canonFromImage(nodes, numNodes, heap, heapBytes, nodesAddr, heapAddr);
}
void canon_destroy(void* h) { delete (Canon*)h; }
int canon_error(void* h) { return ((Canon*)h)->error; }
uint32_t canon_num_nodes(void* h) { return (uint32_t)((Canon*)h)->nodes.size(); }

void canon_records(void* h, CanonRecord* out) {
    Canon& c = *(Canon*)h;
    for (size_t k = 0; k < c.order.size(); k++) {
        const CNode& n = c.nodes[c.order[k]];
        CanonRecord& r = out[k];
        memset(&r, 0, sizeof(r));
        r.level = n.level; r.X = n.X; r.Y = n.Y; r.Z = n.Z; memcpy(r.name, n.name, 20);
        r.counter = n.counter; r.numPoints = n.numPoints; r.numVoxels = n.numVoxels; r.numVoxelsStored = n.numVoxelsStored;
        r.isLeaf = n.isLeaf() ? 1 : 0; r.chunksPoints = n.chunksPoints; r.chunksVoxels = n.chunksVoxels; r.nodeIndex = c.order[k];
        std::vector<Point> pts = n.points; std::sort(pts.begin(), pts.end(), pointLess);
        r.hashPoints = hashBytes(0xcbf29ce484222325ull, pts.data(), pts.size() * 16);
        std::vector<Point> vox = n.voxels; std::sort(vox.begin(), vox.end(), posLess);
        uint64_t hv = 0xcbf29ce484222325ull;
        for (const Point& v : vox) hv = hashBytes(hv, &v, 12);
        r.hashVoxelPos = hv;
    }
}
// sorted samples of the k-th node in canonical order (which: 0 = points, 1 = voxels); returns the count
uint64_t canon_node_samples(void* h, uint32_t k, int which, SimlodPoint* out, uint64_t capacity) {
    Canon& c = *(Canon*)h;
    const CNode& n = c.nodes[c.order[k]];
    std::vector<Point> v = which ? n.voxels : n.points;
    std::sort(v.begin(), v.end(), pointLess);
    uint64_t cnt = std::min<uint64_t>(capacity, v.size());
    if (out) memcpy(out, v.data(), cnt * 16);
    return v.size();
}

// every voxel colour of `other` (same topology as the oracle) must be the colour of a point that
// could have created that voxel: a point of the batch (incl. re-inserted spilled points) in which
// the cell was first occupied. Returns the number of violating voxels, or -1 on a topology mismatch.
int64_t oracle_check_voxel_colors(void* ho, void* hc) {
    Oracle& o = *(Oracle*)ho;
    Canon& c = *(Canon*)hc;
    if (!o.candidatesSorted) { std::sort(o.colorCandidates.begin(), o.colorCandidates.end()); o.candidatesSorted = true; }
    std::map<std::tuple<uint32_t, uint32_t, uint32_t, uint32_t>, int32_t> byKey;
    for (size_t i = 0; i < o.nodes.size(); i++) byKey[{o.nodes[i].level, o.nodes[i].X, o.nodes[i].Y, o.nodes[i].Z}] = (int32_t)i;
    int64_t bad = 0;
    for (const CNode& n : c.nodes) {
        auto it = byKey.find({n.level, n.X, n.Y, n.Z});
        if (it == byKey.end()) return -1;
        const ONode& on = o.nodes[it->second];
        std::unordered_map<uint64_t, uint32_t> cellOfPos;     // voxel position -> cell (positions are unique per cell)
        for (size_t i = 0; i < on.voxels.size(); i++) {
            uint64_t k = 0; memcpy(&k, &on.voxels[i].x, 8);
            uint32_t zbits; memcpy(&zbits, &on.voxels[i].z, 4);
            cellOfPos[k ^ ((uint64_t)zbits * 0x9E3779B97F4A7C15ull)] = on.voxelCells[i];
        }
        for (const Point& v : n.voxels) {
            uint64_t k = 0; memcpy(&k, &v.x, 8);
            uint32_t zbits; memcpy(&zbits, &v.z, 4);
            auto ci = cellOfPos.find(k ^ ((uint64_t)zbits * 0x9E3779B97F4A7C15ull));
            if (ci == cellOfPos.end()) { bad++; continue; }
            std::pair<uint64_t, uint32_t> probe{((uint64_t)it->second << 21) | ci->second, v.color};
            if (!std::binary_search(o.colorCandidates.begin(), o.colorCandidates.end(), probe)) bad++;
        }
    }
    return bad;
}

void canon_render(void* h, const SimlodUniforms* u, uint64_t* fb, RenderStats* rs) { renderCanon(*(Canon*)h, *u, fb, rs); }
// visibility flags of the last canon_render in canonical node order: out[2*k] = visible, out[2*k+1] = isLarge
void canon_flags(void* h, uint8_t* out) {
    Canon& c = *(Canon*)h;
    for (size_t k = 0; k < c.order.size(); k++) { out[2 * k] = c.nodes[c.order[k]].visible; out[2 * k + 1] = c.nodes[c.order[k]].isLarge; }
}

}  // extern "C"

// ---- LAS record decode (SURVEY.md §8f-2): restatement of loadLasNative's parse loop, LasLoader.cpp:176-225 ----
extern "C" void oracle_decode_las(const uint8_t* records, uint64_t numPoints, uint32_t bytesPerPoint, uint32_t format,
                                  const double* scale, const double* offset, const double* translation, SimlodPoint* out) {
    uint64_t offsetRgb = 0;                                   // :179-188
    if (format == 2) offsetRgb = 20; else if (format == 3) offsetRgb = 28;
    if (format == 5) offsetRgb = 28;
    if (format == 7) offsetRgb = 30;
    const double ox = offset[0] + translation[0], oy = offset[1] + translation[1], oz = offset[2] + translation[2];   // :199-201
    for (uint64_t i = 0; i < numPoints; i++) {
        const uint8_t* src = records + bytesPerPoint * i;
        int32_t XYZ[3];
        memcpy(XYZ, src, 12);
        SimlodPoint p;
        volatile double mx = double(XYZ[0]) * scale[0], my = double(XYZ[1]) * scale[1], mz = double(XYZ[2]) * scale[2];   // no contraction
        p.x = (float)(mx + ox); p.y = (float)(my + oy); p.z = (float)(mz + oz);                                            // :206-208
        uint32_t color = 0xff000000u;                         // alpha (and colour without RGB) is uninitialised in the reference: compared under a mask
        if (offsetRgb > 0) {
            uint16_t rgb[3];
            memcpy(rgb, src + offsetRgb, 6);
            uint32_t r = rgb[0] > 255 ? rgb[0] / 256 : rgb[0], g = rgb[1] > 255 ? rgb[1] / 256 : rgb[1], b = rgb[2] > 255 ? rgb[2] / 256 : rgb[2];   // :212-217
            color |= r | (g << 8) | (b << 16);
        }
        p.color = color;
        out[i] = p;
    }
}

// ---- spatial exchange (SURVEY.md §8f-3): the level-`level` octree cell a point descends into, with the builder's
// own quantisation (voxels.cu:148-155) and child order (voxels.cu:171-179); cell = child indices root first.
extern "C" void oracle_partition_cells(const SimlodPoint* pts, uint64_t n, const float* boxMin, const float* boxMax, float rcpSize,
                                       uint32_t level, uint32_t* cells) {
    Quantizer qz;
    qz.minx = boxMin[0]; qz.miny = boxMin[1]; qz.minz = boxMin[2];
    qz.size = std::max(std::max(boxMax[0] - boxMin[0], boxMax[1] - boxMin[1]), boxMax[2] - boxMin[2]);
    qz.rcp = rcpSize;
    for (uint64_t i = 0; i < n; i++) {
        Coords q = qz(pts[i]);
        uint32_t cell = 0;
        for (uint32_t l = 0; l < level; l++) cell = (cell << 3) | childIndexAt(q, (int)l);
        cells[i] = cell;
    }
}
