"""The persistent-heap capacity guard (reference voxels.cu:896-912) on every entry path (run with -m gpu on an H100).

The reference's rule: let H_j be the heap offset (Stats::allocatedBytes_persistent) once batches [0, j) are complete.
Before it consumes batch j, kernel_construct reads that offset after a grid barrier and stops iff
H_j + 200 000 000 >= persistentBufferCapacity; it then raises Stats::memCapacityReached and consumes nothing further.
So a stream of N batches stops after j* = min{ j < N : H_j + 200 MB >= capacity } batches, or after all N.

H_j comes from the CPU oracle (its allocatedBytes_persistent is pinned to the reference kernels in
tests/golden/reference.json). The capacities sit exactly on the edge, C = H_j + 200 MB + delta: with delta = 0 the
reference stops before batch j, with delta = 1 it consumes batch j. Our builder pipelines batches (the chunks of batch
j-1 are allocated while batch j is counted) and launches up to 20 batches at once, so the batches in the middle of a
launch are the ones where the guard can go wrong by a whole batch.
"""
import ctypes

import pytest

import oracle
import reference_golden as golden
from simlod_b200 import SimLOD, SimlodError, camera, data

pytestmark = pytest.mark.gpu

MARGIN = 200_000_000
ERR_CAPACITY = -5


def expected_stop(H, n, capacity):
    """Batches the reference consumes of the first n when the heap holds `capacity` bytes (H[j] = H_j)."""
    return next((j for j in range(n) if H[j] + MARGIN >= capacity), n)


class Stream:
    """A point stream, its batches, and the oracle's octree after any prefix of them. The oracle only moves forward;
    asking for an earlier prefix builds it again."""

    def __init__(self, name, pts, box, batch_size, gen, rcp=0.0):
        self.name, self.pts, self.box, self.gen, self.rcp = name, pts, box, gen, rcp
        self.batches = list(data.batches(pts, batch_size))
        self.sizes = [len(b) for b in self.batches]
        self.n = len(self.batches)
        self._restart()
        self.H = [self._o.stats().allocatedBytes_persistent]
        for b in self.batches:
            self._o.add_batch(b)
            self.H.append(self._o.stats().allocatedBytes_persistent)
        self._at = self.n
        self._cache = {}

    def _restart(self):
        self._o = oracle.Oracle(self.box[0], self.box[1], self.rcp)
        self._at = 0

    def oracle_at(self, j):
        if j < self._at:
            self._restart()
        while self._at < j:
            self._o.add_batch(self.batches[self._at])
            self._at += 1
        return self._o

    def octree(self, j):
        """(Stats, canonical form) of the oracle after j batches."""
        if j not in self._cache:
            o = self.oracle_at(j)
            self._cache[j] = (o.stats(), o.canon())
        return self._cache[j]

    def capacity(self, j, delta):
        return self.H[j] + MARGIN + delta


@pytest.fixture(scope="module")
def streams():
    s = SimLOD(320, 176, persistent_bytes=1 << 30)
    try:
        rcp = float(s.device_rcp(4800.0))      # the terrain cube is 4800 wide: not a power of two, 1/size is the device's
    finally:
        s.close()
    pts, mn, mx = data.terrain(25_654_321)
    # 26 batches: two 20-batch launches on the zero-copy path, a ragged last batch
    a = Stream("terrain26", pts, (mn, mx), 1_000_000, (SimLOD.GEN_TERRAIN, len(pts), 7, 0.0), rcp)
    pts, mn, mx = data.uniform_cube(3_000_000, size=2048.0, seed=77)
    # incoherent: the root and all 8 of its children fill at the same rate and split in batch 0, a cascade of 9 splits
    # whose grids batch 1's guard has to account for (1 M-point batches: the size the C insertion paths cut a stream into)
    b = Stream("uniform3", pts, (mn, mx), 1_000_000, (SimLOD.GEN_UNIFORM, 0, 77, 2048.0))
    return {"terrain26": a, "uniform3": b}


def new_sim(stream, capacity, **kw):
    sim = SimLOD(320, 176, persistent_bytes=capacity, **kw)
    assert sim.uniforms.persistentBufferCapacity == capacity
    sim.set_box(*stream.box)
    sim.reset()
    return sim


def raised_code(fn):
    try:
        fn()
    except SimlodError as e:
        return e.code
    return 0


# ---- entry paths: insert the first n batches of the stream, return the error code (0 = none) ---------------------

def insert_device(sim, stream, n):
    """Zero-copy: the points generated in place on the device, 20-batch launches."""
    count = sum(stream.sizes[:n])
    dptr = sim.device_alloc(count * 16)
    try:
        kind, n_total, seed, size = stream.gen
        sim.generate(kind, dptr, n_total, 0, count, seed, size)
        return raised_code(lambda: sim.insert_device(dptr, count))
    finally:
        sim.synchronize()
        sim.device_free(dptr)


def insert_host_ptr(sim, stream, n):
    """Ring copy from pinned host memory, launched every 2 batches."""
    count = sum(stream.sizes[:n])
    hptr = sim.host_alloc(count * 16)
    try:
        ctypes.memmove(hptr, stream.pts.ctypes.data, count * 16)
        return raised_code(lambda: sim.insert_host_ptr(hptr, count))
    finally:
        sim.synchronize()
        sim.host_free(hptr)


def update_octree(sim, stream, n):
    """The reference host's own pattern: batches uploaded ahead, then update launches until nothing moves."""
    for b in stream.batches[:n]:
        sim.upload_batch(b)
    before = -1
    while True:
        sim.update_octree()
        st = sim.stats()
        if st.memCapacityReached or st.batchletIndex == before:
            return 0
        before = st.batchletIndex


def insert_batches(sim, stream, n):
    """One batch per launch."""
    return raised_code(lambda: sim.insert_batches(stream.batches[:n]))


def insert_simlod_file(sim, stream, n, path):
    data.write_simlod(path, stream.pts[:sum(stream.sizes[:n])], *stream.box)
    return raised_code(lambda: sim.insert_simlod_file(path, loader_threads=4))


def check_against_oracle(sim, stream, n, capacity, code, raises=True):
    j = expected_stop(stream.H, n, capacity)
    st = sim.stats()
    assert code == (ERR_CAPACITY if raises and j < n else 0), (code, j, n)
    assert (st.batchletIndex, st.numPointsProcessed, st.memCapacityReached, st.dbg) == (j, sum(stream.sizes[:j]), int(j < n), 0)
    cn = oracle.canon_from_image(*sim.download_octree())
    o_st, o_cn = stream.octree(j)
    diffs = oracle.compare_canon(cn, o_cn, "ours vs oracle after %d batches" % j) + oracle.compare_stats(st, o_st)
    assert not diffs, "\n".join(diffs)
    assert stream.oracle_at(j).check_voxel_colors(cn) == 0
    return st, cn


# capacities: (stream, j, delta); j = None: everything fits. Ordered by the expected stop, so that the oracle walks each
# stream once. Terrain: j = 20 is the first batch of the second zero-copy launch; 7, 19 and 23 fall inside a launch.
EDGES = ([("terrain26", j, d) for j in (0, 7, 19, 20, 23) for d in (0, 1)] + [("terrain26", None, 1)] +
         [("uniform3", j, d) for j in (1, 2) for d in (0, 1)])
PATHS = {"insert_device": insert_device, "insert_host_ptr": insert_host_ptr, "update_octree": update_octree,
         "insert_batches": insert_batches}
CASES = [(s, j, d, p) for (s, j, d) in EDGES for p in PATHS]


def case_id(case):
    s, j, d, p = case
    return "%s-%s-d%d-%s" % (s, "all" if j is None else "j%d" % j, d, p)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_capacity_guard_stops_where_the_reference_does(streams, case):
    name, j, delta, path = case
    stream = streams[name]
    j = stream.n if j is None else j
    capacity = stream.capacity(j, delta)
    n = min(j + 3, stream.n) if path == "update_octree" else stream.n
    sim = new_sim(stream, capacity)
    try:
        code = PATHS[path](sim, stream, n)
        check_against_oracle(sim, stream, n, capacity, code, raises=path != "update_octree")
    finally:
        sim.close()


@pytest.mark.parametrize("delta", [0, 1])
def test_capacity_guard_on_the_file_streamer(streams, tmp_path, delta):
    stream = streams["terrain26"]
    capacity = stream.capacity(7, delta)
    sim = new_sim(stream, capacity)
    try:
        code = insert_simlod_file(sim, stream, stream.n, str(tmp_path / "terrain26.simlod"))
        check_against_oracle(sim, stream, stream.n, capacity, code)
    finally:
        sim.close()


@pytest.mark.parametrize("j,delta", [(7, 0), (7, 1), (20, 0)])
def test_capacity_guard_vs_reference_kernels(streams, j, delta):
    """The reference's own kernels on the zero-copy path at the same capacity: same error, same octree."""
    stream = streams["terrain26"]
    capacity = stream.capacity(j, delta)
    sim = new_sim(stream, capacity, momentary_bytes=oracle.REF_MOMENTARY_BYTES)

    def build(reference):
        for p in (0, 2):
            sim.use_module(p, oracle.REF_CUBINS[p] if reference else None)
        try:
            sim.set_box(*stream.box)
            sim.reset()
            code = insert_device(sim, stream, stream.n)
            return dict(golden.octree(sim.stats(), oracle.canon_from_image(*sim.download_octree())), error=code)
        finally:
            for p in (0, 2):
                sim.use_module(p, None)
    try:
        ours = build(False)
        ref = golden.reference("capacity/terrain26/j%d/d%d/insert_device" % (j, delta), lambda: build(True))
        golden.assert_same(ours, ref, "ours vs reference kernels")
        assert ref["error"] == (ERR_CAPACITY if expected_stop(stream.H, stream.n, capacity) < stream.n else 0)
    finally:
        sim.close()


@pytest.mark.parametrize("path", ["insert_device", "insert_host_ptr"])
def test_context_works_after_a_capacity_error(streams, path):
    """An insertion that stops on the guard returns with launches still queued; the context must stay usable."""
    stream = streams["terrain26"]
    capacity = stream.capacity(7, 0)
    sim = new_sim(stream, capacity)
    try:
        assert PATHS[path](sim, stream, stream.n) == ERR_CAPACITY
        sim.reset()
        code = PATHS[path](sim, stream, 3)         # a prefix that fits
        check_against_oracle(sim, stream, 3, capacity, code)
        view, proj = camera.autofocus(stream.box[1], sim.width, sim.height)
        sim.set_camera(view, proj)
        sim.render()
        assert sim.stats().numVisibleNodes > 0
    finally:
        sim.close()
