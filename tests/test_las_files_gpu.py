"""simlod_insert_files on the GPU: the octree a file list streams in is the octree of the restated batches
(tests/files_restatement.py: the reference's reload() box, translation and batch list, LAS records decoded by
oracle.decode_las, whose output is pinned against the reference's loadLasNative), inserted one batch at a time;
and a failing call leaves the context as it was."""
import hashlib
import os

import numpy as np
import pytest

import files_restatement as fr
import oracle
from simlod_b200 import SimLOD, SimlodError, data

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(320, 176, persistent_bytes=8 << 30)
    yield s
    s.close()


def octree_of(sim):
    return sim.stats(), oracle.canon_from_image(*sim.download_octree())


def restated_octree(sim, paths, key=None):
    """The octree of reload(paths)'s batches inserted one by one into a reset context with the restated box."""
    restated = fr.check_batches_against_reference(key, paths) if key else fr.reload(paths)
    bmin, bmax, tr, batches = restated
    sim.set_box((0.0, 0.0, 0.0), bmax - bmin)
    sim.reset()
    sim.insert_batches(fr.batch_points(b, tr) for b in batches)
    return octree_of(sim), restated


def assert_files_build_restated_octree(sim, paths, key=None, **kw):
    n, kms, tms = sim.insert_files(paths, **kw)
    st_a, cn_a = octree_of(sim)
    box = [list(sim.uniforms.boxMin), list(sim.uniforms.boxMax)]
    (st_b, cn_b), (bmin, bmax, _, batches) = restated_octree(sim, paths, key)
    assert n == sum(b[2] for b in batches) and st_a.numPointsProcessed == n and st_a.dbg == 0
    assert st_a.batchletIndex == len(batches)
    assert box == [[0.0, 0.0, 0.0], [float(v) for v in (bmax - bmin).astype(np.float32)]]
    diffs = oracle.compare_canon(cn_a, cn_b) + oracle.compare_stats(st_a, st_b)
    assert not diffs, diffs
    return st_a, cn_a, kms, tms


@pytest.mark.parametrize("case", sorted(fr.FORMAT_CASES))
def test_one_las_file_per_format(sim, tmp_path, case):
    path = fr.write_format_case(tmp_path, case)
    _, _, kms, tms = assert_files_build_restated_octree(sim, [path], key="format/" + case)
    assert kms > 0 and tms > 0


def write_tiles(directory):
    """Four 1.2 M-point LAS tiles of one terrain with different formats, scales and offsets, and an empty tile."""
    specs = [(2, (0.001, 0.001, 0.001), (1000.0, 2000.0, 0.0), (1, 2), 0), (3, (0.01, 0.01, 0.01), (0.0, 0.0, 0.0), (1, 4), 54),
             (0, (0.0005, 0.0005, 0.0005), (-3.0, 11.0, 7.0), (1, 3), 0), (7, (0.002, 0.001, 0.004), (900.0, 1900.0, 40.0), (1, 4), 0)]
    n_tile, paths = 1_200_000, []
    for k, (fmt, scale, offset, version, vlr) in enumerate(specs):
        p = os.path.join(str(directory), "tile%d.las" % k)
        data.write_las(p, fr.shifted_terrain(4 * n_tile, k * n_tile, n_tile), fmt=fmt, scale=scale, offset=offset, version=version, vlr_bytes=vlr)
        paths.append(p)
    empty = os.path.join(str(directory), "empty.las")
    data.write_las(empty, np.zeros(0, dtype=oracle.POINT_DTYPE), fmt=2)
    return paths, empty


def test_lists_of_tiles_and_mixed_lists(sim, tmp_path):
    tiles, empty = write_tiles(tmp_path)
    assert_files_build_restated_octree(sim, tiles)
    # an empty tile adds its (zero) box and no batch
    assert_files_build_restated_octree(sim, [tiles[0], empty, tiles[2]])
    # .simlod points are inserted untranslated beside translated LAS records
    sml = str(tmp_path / "part.simlod")
    pts, mn, mx = data.terrain(1_500_000)
    data.write_simlod(sml, pts, mn, mx)
    assert_files_build_restated_octree(sim, [sml, tiles[1]])


def test_loader_thread_counts_and_the_one_simlod_file_case(sim, tmp_path):
    tiles, _ = write_tiles(tmp_path)
    _, cn_1, _, _ = assert_files_build_restated_octree(sim, tiles, loader_threads=1)
    for threads in (4, 16):
        sim.insert_files(tiles, loader_threads=threads)
        _, cn = octree_of(sim)
        assert not oracle.compare_canon(cn, cn_1), threads
    sml = str(tmp_path / "scan.simlod")
    pts, mn, mx = data.terrain(2_300_017)
    data.write_simlod(sml, pts, mn, mx)
    sim.insert_simlod_file(sml)
    st_a, cn_a = octree_of(sim)
    box_a = bytes(sim.uniforms)[424:448]
    sim.insert_files([sml])
    st_b, cn_b = octree_of(sim)
    assert bytes(sim.uniforms)[424:448] == box_a
    assert not oracle.compare_canon(cn_a, cn_b) and not oracle.compare_stats(st_a, st_b)


def test_unbuffered_reads(sim, tmp_path):
    """direct=True (O_DIRECT, any offset_to_point_data): the same octree. Skipped where the file system cannot do
    O_DIRECT (tmpfs)."""
    tiles, _ = write_tiles(tmp_path)
    for p in tiles:
        fd = os.open(p, os.O_RDONLY)
        try:
            os.fsync(fd)
            os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
        finally:
            os.close(fd)
    try:
        assert_files_build_restated_octree(sim, tiles, loader_threads=5, direct=True)
    except SimlodError as e:
        if "O_DIRECT" in str(e):
            pytest.skip("file system of %s does not support O_DIRECT" % tmp_path)
        raise


def context_digest(sim):
    nodes, heap, _, _ = sim.download_octree()
    b = sim.buffers()
    raw_stats = sim.memcpy_dtoh(b.stats, 112)
    return hashlib.sha256(nodes.tobytes() + raw_stats.tobytes() + bytes(sim.uniforms)).hexdigest(), heap.nbytes


def test_a_failing_call_leaves_the_context_unchanged(sim, tmp_path):
    tiles, _ = write_tiles(tmp_path)
    sim.insert_files(tiles[:2])
    before = context_digest(sim)
    bad = tmp_path / "bad.las"
    bad.write_bytes(open(tiles[3], "rb").read()[:-7])
    laz = tmp_path / "x.laz"
    laz.write_bytes(open(tiles[3], "rb").read()[:4096])
    for paths in ([], [tiles[0], str(tmp_path / "missing.las")], [tiles[0], str(bad)], [str(laz)], [tiles[1], str(tmp_path)]):
        with pytest.raises(SimlodError) as e:
            sim.insert_files(paths)
        assert e.value.code == -2
        assert context_digest(sim) == before, paths


def test_full_size_one_file_and_eight_tiles(tmp_path):
    """36 M terrain points as one LAS format 3 file (1.2 GB) and as 8 format 2 tiles: both give the octree of the
    decoded points, batch for batch."""
    n = 36_000_000
    sim = SimLOD(320, 176, persistent_bytes=8 << 30)
    try:
        dptr = sim.device_alloc(n * 16)
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        pts = sim.memcpy_dtoh(dptr, n * 16).view(oracle.POINT_DTYPE)
        sim.device_free(dptr)
        one = str(tmp_path / "scan.las")
        data.write_las(one, pts, fmt=3, scale=(0.001, 0.001, 0.001))
        tiles = []
        for k in range(8):
            p = str(tmp_path / ("tile%d.las" % k))
            data.write_las(p, pts[k * n // 8:(k + 1) * n // 8], fmt=2, scale=(0.001, 0.001, 0.001))
            tiles.append(p)
        del pts
        for paths in ([one], tiles):
            got_n, kms, tms = sim.insert_files(paths)
            st_a, cn_a = octree_of(sim)
            assert got_n == n and st_a.numPointsProcessed == n and st_a.dbg == 0
            bmin, bmax, tr, batches = fr.reload(paths)
            sim.set_box((0.0, 0.0, 0.0), bmax - bmin)
            sim.reset()
            sim.insert_batches(fr.batch_points(b, tr) for b in batches)
            st_b, cn_b = octree_of(sim)
            diffs = oracle.compare_canon(cn_a, cn_b) + oracle.compare_stats(st_a, st_b)
            assert not diffs, (len(paths), diffs)
            print("%d file(s): %d points, kernel %.1f ms, total %.1f ms" % (len(paths), n, kms, tms))
    finally:
        sim.close()
