"""ctypes binding of include/simlod_b200.h and the `SimLOD` host object.

`SimLOD` mirrors the reference's host functions one to one (same names in snake case, same
argument meaning, same error behaviour: launch errors are reported, device-side conditions are
observed through Stats):

    reference (main_progressive_octree.cpp)        here
    initCuda + initCudaProgram   :272, :549         SimLOD(width, height, ...)
    getUniforms                  :283               set_camera / set_box / settings -> uniforms
    resetCUDA                    :333               reset()
    uploader step                :1033-1056         upload_batch()
    updateOctree                 :364               update_octree()
    renderCUDA                   :465               render()
    stats read-back              :1201              stats()

There is no fallback: if libsimlod_b200.so is missing or no H100 is present, construction raises.
"""
import contextlib
import ctypes as C
import math
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsimlod_b200.so")

POINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("color", "<u4")])
# SimlodExportNode (include/simlod_abi.h), 64 bytes
EXPORT_NODE_DTYPE = np.dtype([
    ("level", "<u4"), ("X", "<u4"), ("Y", "<u4"), ("Z", "<u4"), ("name", "S20"), ("flags", "<u4"),
    ("parent", "<i4"), ("first_child", "<i4"), ("sample_offset", "<u8"), ("num_points", "<u4"), ("num_voxels", "<u4")])
EXPORT_LEAF, EXPORT_SAMPLED = 1, 2

MAX_BATCH_SIZE = 1_000_000
BATCH_STREAM_SIZE = 50
FB_OFFSET = 31_200_144
NODE_BYTES = 152
CHUNK_STRIDE = 16032
GRID_STRIDE = 262160

PROGRAM_CONSTRUCT, PROGRAM_RENDER, PROGRAM_RESET = 0, 1, 2


class SimlodError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("simlod_b200 error %d: %s" % (code, message))
        self.code = code


class Float4(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("z", C.c_float), ("w", C.c_float)]


class Mat4(C.Structure):
    _fields_ = [("rows", Float4 * 4)]


class Uniforms(C.Structure):
    """HostDeviceInterface.h:10-44, 480 bytes."""
    _fields_ = [
        ("width", C.c_float), ("height", C.c_float), ("time", C.c_float), ("fovy_rad", C.c_float),
        ("world", Mat4), ("view", Mat4), ("proj", Mat4), ("transform", Mat4),
        ("transform_updateBound", Mat4), ("transformInv_updateBound", Mat4),
        ("persistentBufferCapacity", C.c_uint64), ("momentaryBufferCapacity", C.c_uint64), ("frameCounter", C.c_uint64),
        ("boxMin", C.c_float * 3), ("boxMax", C.c_float * 3),
        ("showBoundingBox", C.c_uint8), ("showPoints", C.c_uint8), ("colorByNode", C.c_uint8), ("colorByLOD", C.c_uint8),
        ("colorWhite", C.c_uint8), ("doUpdateVisibility", C.c_uint8), ("doProgressive", C.c_uint8), ("_pad0", C.c_uint8),
        ("LOD", C.c_float),
        ("useHighQualityShading", C.c_uint8), ("_pad1", C.c_uint8 * 3),
        ("minNodeSize", C.c_float), ("pointSize", C.c_int32),
        ("updateStats", C.c_uint8), ("enableEDL", C.c_uint8), ("_pad2", C.c_uint8 * 2),
        ("edlStrength", C.c_float),
    ]


class Stats(C.Structure):
    """HostDeviceInterface.h:46-71, 112 bytes."""
    _fields_ = [
        ("frameID", C.c_uint32), ("numNodes", C.c_uint32), ("numInner", C.c_uint32), ("numLeaves", C.c_uint32),
        ("numNonemptyLeaves", C.c_uint32), ("numPoints", C.c_uint32), ("numVoxels", C.c_uint32), ("_pad0", C.c_uint32),
        ("allocatedBytes_momentary", C.c_uint64), ("allocatedBytes_persistent", C.c_uint64),
        ("numVisibleNodes", C.c_uint32), ("numVisibleInner", C.c_uint32), ("numVisibleLeaves", C.c_uint32),
        ("numVisiblePoints", C.c_uint32), ("numVisibleVoxels", C.c_uint32), ("numChunksPoints", C.c_uint32),
        ("numChunksVoxels", C.c_uint32), ("batchletIndex", C.c_uint32),
        ("numPointsProcessed", C.c_uint64), ("numAllocatedChunks", C.c_uint64), ("chunkPoolSize", C.c_uint64),
        ("dbg", C.c_uint32), ("memCapacityReached", C.c_uint8), ("_pad1", C.c_uint8 * 3),
    ]


class Config(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("width", C.c_uint32), ("height", C.c_uint32),
        ("momentary_bytes", C.c_uint64), ("nodes_bytes", C.c_uint64), ("renderbuffer_bytes", C.c_uint64),
        ("persistent_bytes", C.c_uint64), ("construct_blocks_per_sm", C.c_int32), ("render_blocks_per_sm", C.c_int32),
    ]


class LasLayout(C.Structure):
    _fields_ = [("bytes_per_point", C.c_uint32), ("format", C.c_uint32), ("scale", C.c_double * 3), ("offset", C.c_double * 3),
                ("translation", C.c_double * 3)]


class LasHeader(C.Structure):
    """SimlodLasHeader: the LAS public header fields the reference reads (LasLoader.h:21-55), 128 bytes."""
    _fields_ = [("version_major", C.c_uint32), ("version_minor", C.c_uint32), ("format", C.c_uint32), ("bytes_per_point", C.c_uint32),
                ("header_size", C.c_uint32), ("offset_to_point_data", C.c_uint32), ("num_points", C.c_uint64),
                ("scale", C.c_double * 3), ("offset", C.c_double * 3), ("min", C.c_double * 3), ("max", C.c_double * 3)]

    def as_dict(self):
        return {f: (tuple(getattr(self, f)) if f in ("scale", "offset", "min", "max") else int(getattr(self, f))) for f, _ in self._fields_}


class PartitionPlan(C.Structure):
    """SimlodPartitionPlan: the level-`level` cells of the octree cube and the rank that owns each."""
    _fields_ = [("level", C.c_uint32), ("num_ranks", C.c_uint32), ("owner", C.c_uint8 * 512)]


class Buffers(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "nodes", "nodes_bytes", "persistent", "persistent_bytes", "momentary", "momentary_bytes",
        "renderbuffer", "renderbuffer_bytes", "ring", "ring_bytes", "stats")]


class ExportInfo(C.Structure):
    """SimlodExportInfo: records in the export, deepest level in the octree, sample counts."""
    _fields_ = [("num_nodes", C.c_uint32), ("max_level", C.c_uint32), ("num_samples", C.c_uint64), ("num_points", C.c_uint64),
                ("num_voxels", C.c_uint64)]


class OctreeFileHeader(C.Structure):
    """SimlodOctreeFileHeader: the 128-byte header of an octree file (SimLOD.save_octree), format version 1."""
    _fields_ = [("magic", C.c_char * 8), ("version", C.c_uint32), ("header_size", C.c_uint32), ("info", ExportInfo),
                ("box_min", C.c_float * 3), ("box_max", C.c_float * 3), ("batchlet_index", C.c_uint32), ("reserved0", C.c_uint32),
                ("num_points_processed", C.c_uint64), ("records_offset", C.c_uint64), ("counters_offset", C.c_uint64),
                ("samples_offset", C.c_uint64), ("file_size", C.c_uint64), ("reserved1", C.c_uint64)]


REGION_BOX, REGION_SPHERE, REGION_PLANES = 1, 2, 3
REGION_MAX_PLANES = 16


class SimlodRegion(C.Structure):
    """SimlodRegion: a box, a sphere or up to 16 half-spaces, in the coordinates of the stored samples."""
    _fields_ = [("kind", C.c_uint32), ("num_planes", C.c_uint32), ("box_min", C.c_float * 3), ("box_max", C.c_float * 3),
                ("center", C.c_float * 3), ("radius", C.c_float), ("planes", (C.c_float * 4) * REGION_MAX_PLANES)]


CLIP_NONE, CLIP_INSIDE, CLIP_OUTSIDE = 0, 1, 2
CLIP_MAX_REGIONS = 4


class SimlodClip(C.Structure):
    """SimlodClip: render() and pick() draw only the samples inside (INSIDE) or outside (OUTSIDE) the union of the first
    num_regions regions."""
    _fields_ = [("mode", C.c_uint32), ("num_regions", C.c_uint32), ("regions", SimlodRegion * CLIP_MAX_REGIONS)]


class SimlodQueryInfo(C.Structure):
    """SimlodQueryInfo: what a region query returned and how much of the octree it had to look at."""
    _fields_ = [("num_samples", C.c_uint64), ("num_points", C.c_uint64), ("num_voxels", C.c_uint64), ("samples_tested", C.c_uint64),
                ("nodes_visited", C.c_uint32), ("max_level", C.c_uint32)]


class SimlodPickInfo(C.Structure):
    """SimlodPickInfo: hits among the requested pixels, the view export's sample and record counts (the index space), and
    the event time of each stage of the pick."""
    _fields_ = [("num_hits", C.c_uint64), ("num_samples", C.c_uint64), ("num_nodes", C.c_uint32), ("num_pixels", C.c_uint32),
                ("plan_ms", C.c_float), ("key_ms", C.c_float), ("index_ms", C.c_float), ("write_ms", C.c_float)]


NEAREST_MAX_K = 32
NEAREST_MAX_QUERIES = 1 << 24


class SimlodNearestInfo(C.Structure):
    """SimlodNearestInfo: the export's sample count (the index space), filled slots, how much of the octree the search
    had to look at, and the event time of each stage."""
    _fields_ = [("num_samples", C.c_uint64), ("num_found", C.c_uint64), ("samples_tested", C.c_uint64),
                ("records_visited", C.c_uint64), ("num_queries", C.c_uint32), ("k", C.c_uint32), ("invalid_queries", C.c_uint32),
                ("max_level", C.c_uint32), ("plan_ms", C.c_float), ("bucket_ms", C.c_float), ("search_ms", C.c_float),
                ("reserved", C.c_uint32)]


RAY_MAX_RAYS = 1 << 24


class SimlodRayInfo(C.Structure):
    """SimlodRayInfo: the export's sample count (the index space), rays with a hit, how much of the octree the trace had
    to look at, and the event time of each stage."""
    _fields_ = [("num_samples", C.c_uint64), ("num_hits", C.c_uint64), ("samples_tested", C.c_uint64),
                ("records_visited", C.c_uint64), ("num_rays", C.c_uint32), ("invalid_rays", C.c_uint32),
                ("max_level", C.c_uint32), ("plan_ms", C.c_float), ("trace_ms", C.c_float), ("reserved", C.c_uint32)]


RADIUS_MAX_QUERIES = 1 << 24


class SimlodRadiusInfo(C.Structure):
    """SimlodRadiusInfo: the export's sample count (the index space), the neighbours found (offsets[-1]), how much of the
    octree the count pass had to look at, the largest neighbourhood, and the event time of each stage."""
    _fields_ = [("num_samples", C.c_uint64), ("num_found", C.c_uint64), ("samples_tested", C.c_uint64),
                ("records_visited", C.c_uint64), ("num_queries", C.c_uint32), ("invalid_queries", C.c_uint32),
                ("max_level", C.c_uint32), ("max_found", C.c_uint32), ("plan_ms", C.c_float), ("bucket_ms", C.c_float),
                ("count_ms", C.c_float), ("write_ms", C.c_float)]


HEIGHTMAP_MAX_CELLS = 1 << 27


class SimlodHeightmap(C.Structure):
    """SimlodHeightmap: a grid of nx x ny square cells of edge `cell` over the x-y plane, cell (0, 0) at `origin`."""
    _fields_ = [("origin", C.c_float * 2), ("cell", C.c_float), ("nx", C.c_uint32), ("ny", C.c_uint32), ("reserved", C.c_uint32)]


class SimlodHeightmapInfo(C.Structure):
    """SimlodHeightmapInfo: the export's sample count (the index space), the samples binned (the sum of the counts), how
    much of the octree the culling left to read, the non-empty cells, and the event time of each stage."""
    _fields_ = [("num_samples", C.c_uint64), ("num_binned", C.c_uint64), ("samples_tested", C.c_uint64),
                ("records_visited", C.c_uint64), ("nonempty_cells", C.c_uint64), ("max_level", C.c_uint32),
                ("plan_ms", C.c_float), ("accumulate_ms", C.c_float), ("finalize_ms", C.c_float)]


class LasWriteParams(C.Structure):
    """SimlodLasWriteParams: the file's scale and offset, the translation added to every sample, the writer threads."""
    _fields_ = [("scale", C.c_double * 3), ("offset", C.c_double * 3), ("translation", C.c_double * 3),
                ("writer_threads", C.c_uint32), ("reserved", C.c_uint32)]


class LasWriteInfo(C.Structure):
    """SimlodLasWriteInfo: records written, file size, the first invalid sample (UINT64_MAX for none), the header's
    bounds, and the time of each stage."""
    _fields_ = [("num_points", C.c_uint64), ("file_size", C.c_uint64), ("first_invalid", C.c_uint64),
                ("min", C.c_double * 3), ("max", C.c_double * 3), ("plan_ms", C.c_float), ("encode_ms", C.c_float),
                ("copy_ms", C.c_float), ("write_ms", C.c_float), ("num_windows", C.c_uint32), ("reserved", C.c_uint32)]


NO_INVALID = (1 << 64) - 1


class Region:
    """Constructors of the regions SimLOD.query_region takes. Numbers are rounded to float32, the type the predicates are
    evaluated in; a malformed region (non-finite number, min > max, negative radius) is refused by the query."""

    @staticmethod
    def box(mn, mx):
        """min <= p <= max on every axis."""
        r = SimlodRegion(kind=REGION_BOX)
        r.box_min[:] = [float(v) for v in mn]
        r.box_max[:] = [float(v) for v in mx]
        return r

    @staticmethod
    def sphere(center, radius):
        """|p - center|^2 <= radius^2."""
        r = SimlodRegion(kind=REGION_SPHERE, radius=float(radius))
        r.center[:] = [float(v) for v in center]
        return r

    @staticmethod
    def planes(planes):
        """n.p + d >= 0 for every row (nx, ny, nz, d) of a (k, 4) array, 1 <= k <= 16; rows are used as given."""
        a = np.asarray(planes, dtype=np.float32)
        if a.ndim != 2 or a.shape[1] != 4 or not 1 <= a.shape[0] <= REGION_MAX_PLANES:
            raise ValueError("planes must be a (k, 4) array with 1 <= k <= %d" % REGION_MAX_PLANES)
        r = SimlodRegion(kind=REGION_PLANES, num_planes=a.shape[0])
        for k in range(a.shape[0]):
            r.planes[k][:] = [float(v) for v in a[k]]
        return r


class OctreeExport:
    """SimLOD.export_octree() / export_view(): `nodes` (EXPORT_NODE_DTYPE records, breadth-first), `samples` (the sample
    array), `info`."""

    def __init__(self, nodes, samples, info):
        self.nodes, self.samples, self.info = nodes, samples, info


assert C.sizeof(Uniforms) == 480 and C.sizeof(Stats) == 112
assert C.sizeof(ExportInfo) == 32 and EXPORT_NODE_DTYPE.itemsize == 64
assert C.sizeof(LasHeader) == 128
assert C.sizeof(OctreeFileHeader) == 128
assert C.sizeof(SimlodRegion) == 304 and C.sizeof(SimlodQueryInfo) == 40
assert C.sizeof(SimlodClip) == 1224 and SimlodClip.regions.offset == 8
assert C.sizeof(SimlodPickInfo) == 40 and C.sizeof(SimlodNearestInfo) == 64 and C.sizeof(SimlodRayInfo) == 56
assert C.sizeof(SimlodRadiusInfo) == 64
assert C.sizeof(SimlodHeightmap) == 24 and C.sizeof(SimlodHeightmapInfo) == 56
assert C.sizeof(LasWriteParams) == 80 and C.sizeof(LasWriteInfo) == 96

# every symbol include/simlod_b200.h declares
EXPORTS = [
    "simlod_create", "simlod_destroy", "simlod_last_error", "simlod_use_module", "simlod_set_uniforms",
    "simlod_get_uniforms", "simlod_reset", "simlod_upload_batch", "simlod_upload_batch_device",
    "simlod_upload_batch_las", "simlod_upload_batch_las_device", "simlod_insert_simlod_file", "simlod_update_octree", "simlod_insert", "simlod_insert_device", "simlod_render", "simlod_get_stats",
    "simlod_read_framebuffer", "simlod_read_surface", "simlod_get_buffers", "simlod_memcpy_dtoh",
    "simlod_memcpy_htod", "simlod_host_alloc", "simlod_host_free", "simlod_device_alloc", "simlod_device_free",
    "simlod_get_launch_info", "simlod_device_rcp", "simlod_synchronize", "simlod_flush_l2",
    "simlod_partition_count", "simlod_partition_scatter", "simlod_partition_wait",
    "simlod_export_framebuffer", "simlod_peer_signal", "simlod_composite_framebuffers", "simlod_generate", "simlod_reset_with_grid", "simlod_insert_simlod_file_ex", "simlod_get_numa_node",
    "simlod_export_octree", "simlod_export_view", "simlod_read_las_header", "simlod_insert_files",
    "simlod_read_octree_header", "simlod_save_octree", "simlod_load_octree", "simlod_query_region",
    "simlod_pick", "simlod_query_nearest", "simlod_query_ray", "simlod_query_radius", "simlod_write_las", "simlod_files_box",
    "simlod_query_heightmap", "simlod_set_clip",
]

_lib = None


def load_library():
    """Load the C-ABI library. Raises if it has not been built: there is no Python fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SimlodError(-4, "%s is missing; run `python -c 'import __graft_entry__ as g; g.build()'`" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.simlod_last_error.restype = C.c_char_p
    vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
    sig = {
        "simlod_create": [C.POINTER(Config), C.POINTER(vp)],
        "simlod_destroy": [vp],
        "simlod_use_module": [vp, C.c_int, C.c_char_p],
        "simlod_set_uniforms": [vp, C.POINTER(Uniforms)],
        "simlod_get_uniforms": [vp, C.POINTER(Uniforms)],
        "simlod_reset": [vp],
        "simlod_reset_with_grid": [vp, u32, u32],
        "simlod_upload_batch": [vp, vp, u32],
        "simlod_upload_batch_device": [vp, u64, u32],
        "simlod_upload_batch_las": [vp, vp, u32, C.POINTER(LasLayout)],
        "simlod_upload_batch_las_device": [vp, u64, u32, C.POINTER(LasLayout)],
        "simlod_insert_simlod_file": [vp, C.c_char_p, C.c_int, C.POINTER(u64), C.POINTER(C.c_float), C.POINTER(C.c_float)],
        "simlod_insert_simlod_file_ex": [vp, C.c_char_p, C.c_int, u32, C.POINTER(u64), C.POINTER(C.c_float), C.POINTER(C.c_float)],
        "simlod_update_octree": [vp, C.POINTER(C.c_float)],
        "simlod_insert": [vp, vp, u64, C.POINTER(C.c_float), C.POINTER(C.c_float)],
        "simlod_insert_device": [vp, u64, u64, C.POINTER(C.c_float), C.POINTER(C.c_float)],
        "simlod_render": [vp, C.POINTER(C.c_float)],
        "simlod_get_stats": [vp, C.POINTER(Stats)],
        "simlod_read_framebuffer": [vp, vp],
        "simlod_read_surface": [vp, vp],
        "simlod_get_buffers": [vp, C.POINTER(Buffers)],
        "simlod_memcpy_dtoh": [vp, vp, u64, u64],
        "simlod_memcpy_htod": [vp, u64, vp, u64],
        "simlod_host_alloc": [vp, u64, C.POINTER(vp)],
        "simlod_host_free": [vp, vp],
        "simlod_device_alloc": [vp, u64, C.POINTER(u64)],
        "simlod_device_free": [vp, u64],
        "simlod_get_launch_info": [vp, C.POINTER(u64), C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)],
        "simlod_device_rcp": [vp, C.c_float, C.POINTER(C.c_float)],
        "simlod_flush_l2": [vp],
        "simlod_get_numa_node": [vp, C.POINTER(C.c_int)],
        "simlod_generate": [vp, C.c_int, u64, u64, u64, u64, C.c_float, u64],
        "simlod_synchronize": [vp],
        "simlod_partition_count": [vp, u64, u32, C.POINTER(PartitionPlan), C.POINTER(u64), C.POINTER(u64)],
        "simlod_partition_scatter": [vp, u64, u32, C.POINTER(PartitionPlan), C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), u32],
        "simlod_partition_wait": [vp, u64, u32, u32, u32],
        "simlod_export_framebuffer": [vp, u64],
        "simlod_peer_signal": [vp, C.POINTER(u64), u32, u32],
        "simlod_composite_framebuffers": [vp, C.POINTER(u64), u32, u32, C.POINTER(u64), u32],
        "simlod_export_octree": [vp, C.c_int32, u64, u64, u64, u64, C.POINTER(ExportInfo), C.POINTER(C.c_float)],
        "simlod_export_view": [vp, u64, u64, u64, u64, C.POINTER(ExportInfo), C.POINTER(C.c_float)],
        "simlod_read_las_header": [C.c_char_p, C.POINTER(LasHeader)],
        "simlod_insert_files": [vp, C.POINTER(C.c_char_p), u32, C.c_int, u32, C.POINTER(u64), C.POINTER(C.c_float), C.POINTER(C.c_float)],
        "simlod_read_octree_header": [C.c_char_p, C.POINTER(OctreeFileHeader)],
        "simlod_save_octree": [vp, C.c_char_p, C.POINTER(ExportInfo), C.POINTER(C.c_float)],
        "simlod_load_octree": [vp, C.c_char_p, C.c_int, C.POINTER(ExportInfo), C.POINTER(C.c_float)],
        "simlod_query_region": [vp, C.POINTER(SimlodRegion), C.c_int32, u64, u64, C.POINTER(SimlodQueryInfo), C.POINTER(C.c_float)],
        "simlod_set_clip": [vp, C.POINTER(SimlodClip)],
        "simlod_pick": [vp, C.POINTER(C.c_uint32), u64, u64, u64, C.POINTER(SimlodPickInfo), C.POINTER(C.c_float)],
        "simlod_query_nearest": [vp, u64, u64, u32, C.c_int32, C.c_float, u64, u64, u64, C.POINTER(SimlodNearestInfo),
                                 C.POINTER(C.c_float)],
        "simlod_query_ray": [vp, u64, u64, C.c_float, C.c_int32, u64, u64, u64, u64, C.POINTER(SimlodRayInfo), C.POINTER(C.c_float)],
        "simlod_query_radius": [vp, u64, u64, C.c_float, C.c_int32, u64, u64, u64, u64, u64, C.POINTER(SimlodRadiusInfo),
                                C.POINTER(C.c_float)],
        "simlod_write_las": [vp, C.c_char_p, C.POINTER(LasWriteParams), u64, u64, C.c_int32, C.POINTER(LasWriteInfo),
                             C.POINTER(C.c_float)],
        "simlod_files_box": [C.POINTER(C.c_char_p), u32, C.POINTER(C.c_float), C.POINTER(C.c_float)],
        "simlod_query_heightmap": [vp, C.POINTER(SimlodHeightmap), C.c_int32, u64, u64, u64, u64, u64, u64,
                                   C.POINTER(SimlodHeightmapInfo), C.POINTER(C.c_float)],
    }
    for name, argtypes in sig.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = None if name == "simlod_destroy" else C.c_int
    _lib = lib
    return lib


def read_las_header(path):
    """The header fields of a LAS file as the reference's loadHeader reads them (simlod_read_las_header): a LasHeader
    (`.as_dict()` for a plain dict). Needs no GPU. Raises SimlodError(-2) naming the file when it is not a LAS file."""
    lib = load_library()
    h = LasHeader()
    rc = lib.simlod_read_las_header(os.fsencode(path), C.byref(h))
    if rc != 0:
        raise SimlodError(rc, lib.simlod_last_error().decode())
    return h


def read_octree_header(path):
    """The header of an octree file (simlod_read_octree_header), checked against itself and the file size: an
    OctreeFileHeader. Needs no GPU. Raises SimlodError(-2) naming the file when it is not a valid octree file."""
    lib = load_library()
    h = OctreeFileHeader()
    rc = lib.simlod_read_octree_header(os.fsencode(path), C.byref(h))
    if rc != 0:
        raise SimlodError(rc, lib.simlod_last_error().decode())
    return h


def files_box(paths):
    """The union box (box_min, box_max) of a list of .las / .simlod files, as SimLOD.insert_files computes it from their
    headers (simlod_files_box), with the same validation and errors. insert_files stores a point at world - box_min, so
    write_las(..., translation=box_min) puts an octree built from the list back at its world position. Needs no GPU."""
    lib = load_library()
    enc = [os.fsencode(p) for p in paths]
    arr = (C.c_char_p * max(1, len(enc)))(*enc)
    mn, mx = (C.c_float * 3)(), (C.c_float * 3)()
    rc = lib.simlod_files_box(arr, len(enc), mn, mx)
    if rc != 0:
        raise SimlodError(rc, lib.simlod_last_error().decode())
    return np.array(mn[:], dtype=np.float32), np.array(mx[:], dtype=np.float32)


def las_write_params(scale=0.001, offset=None, translation=(0.0, 0.0, 0.0), writer_threads=8):
    """SimlodLasWriteParams from a scalar or 3-tuple scale, an offset (None: the translation) and a translation."""
    sc = [float(scale)] * 3 if np.ndim(scale) == 0 else [float(v) for v in scale]
    tr = [float(v) for v in translation]
    of = tr if offset is None else [float(v) for v in offset]
    if len(sc) != 3 or len(tr) != 3 or len(of) != 3:
        raise ValueError("scale, offset and translation take 3 values (a scalar scale applies to every axis)")
    p = LasWriteParams(writer_threads=int(writer_threads))
    p.scale[:], p.offset[:], p.translation[:] = sc, of, tr
    return p


def make_points(xyz, color):
    """Pack float32 xyz (N,3) and uint32 colours (N,) into the 16-byte reference Point layout."""
    xyz = np.asarray(xyz, dtype=np.float32)
    pts = np.empty(xyz.shape[0], dtype=POINT_DTYPE)
    pts["x"], pts["y"], pts["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    pts["color"] = np.asarray(color, dtype=np.uint32)
    return pts


def _as_points(points):
    a = np.ascontiguousarray(points)
    if a.dtype != POINT_DTYPE:
        if a.dtype.itemsize * (a.shape[-1] if a.ndim > 1 else 1) != 16:
            raise ValueError("points must be 16-byte XYZRGBA records")
        a = a.reshape(-1).view(POINT_DTYPE) if a.ndim == 1 else a.view(POINT_DTYPE).reshape(-1)
    return a


I8, F4 = np.dtype(np.int64), np.dtype(np.float32)
# numpy dtype of a destination -> (torch dtype, trailing shape) of the tensor that holds it on a CUDA device
_TORCH_DESTS = {I8: ("int64", ()), F4: ("float32", ()), POINT_DTYPE: ("float32", (4,))}


class _Results:
    """The destinations of one call on `device`, one per (shape, dtype) in `dests` (dtype I8, F4, POINT_DTYPE or
    EXPORT_NODE_DTYPE; None for one the call does not write). `ptrs` holds their device addresses: 0 for None and for a
    destination without elements, unless `keep`, which gives each destination at least one row. device="cpu": device
    memory, freed when the `with` block ends. A CUDA device: torch tensors, and one synchronisation of torch's stream
    once they are allocated, since the caching allocator may hand out memory torch still uses. results() returns the
    destinations that are not None, `shape` each: numpy arrays copied out of the device memory, or the tensors
    (EXPORT_NODE_DTYPE as a numpy array)."""
    __slots__ = ("_sim", "_dests", "_bufs", "ptrs")

    def __init__(self, sim, device, dests, keep=False):
        self._sim, self._dests, self._bufs, self.ptrs = sim, dests, None, [0] * len(dests)
        if device == "cpu":
            try:
                for i, d in enumerate(dests):
                    if d is not None:
                        nbytes = (max(d[0][0], 1) if keep else d[0][0]) * math.prod(d[0][1:]) * d[1].itemsize
                        if nbytes:
                            self.ptrs[i] = sim.device_alloc(nbytes)
            except BaseException:
                self.__exit__()
                raise
            return
        import torch
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("device must be 'cpu' or a CUDA device, not %r" % device)
        if dev.index is None:
            dev = torch.device("cuda", sim.device)
        bufs = self._bufs = [None] * len(dests)
        for i, d in enumerate(dests):
            if d is not None:
                shape, t = d
                rows = max(shape[0], 1) if keep else shape[0]
                kind = _TORCH_DESTS.get(t)
                bufs[i] = (torch.empty((rows,) + shape[1:] + kind[1], dtype=getattr(torch, kind[0]), device=dev) if kind else
                           torch.empty(rows * t.itemsize, dtype=torch.uint8, device=dev))
        torch.cuda.current_stream(dev).synchronize()
        self.ptrs = [b.data_ptr() if b is not None and b.numel() else 0 for b in bufs]

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        if self._bufs is None:
            for p in self.ptrs:
                if p:
                    self._sim.device_free(p)

    def results(self):
        out = []
        for i, d in enumerate(self._dests):
            if d is None:
                continue
            shape, t = d
            if self._bufs is None:
                out.append(self._sim.memcpy_dtoh(self.ptrs[i], math.prod(shape) * t.itemsize).view(t).reshape(shape))
            elif t not in _TORCH_DESTS:
                out.append(self._bufs[i].cpu().numpy().view(t))
            else:
                b = self._bufs[i]
                out.append(b if b.shape[0] == shape[0] else b[:shape[0]])
        return tuple(out)


class _DeviceInput:
    """An (N, W) float32 array at a 16-byte aligned device address (`ptr`) for the `with` block. A numpy array is copied
    into device memory freed when the block ends (an empty one still gets an address); a CUDA tensor is used in place
    when it is contiguous and 16-byte aligned, else copied, and torch's stream is synchronised, since the tensor may
    still be being computed."""
    __slots__ = ("_sim", "_keep", "ptr")

    def __init__(self, sim, a):
        self._sim = sim
        if isinstance(a, np.ndarray):
            self._keep, self.ptr = None, sim.device_alloc(max(a.nbytes, 16))
            if a.nbytes:
                try:
                    sim.memcpy_htod(self.ptr, a)
                except BaseException:
                    sim.device_free(self.ptr)
                    raise
            return
        import torch
        if not a.is_contiguous() or a.data_ptr() % 16:
            a = a.contiguous().clone()
        torch.cuda.current_stream(a.device).synchronize()
        self._keep, self.ptr = a, a.data_ptr()                # the tensor stays alive until the block ends

    def __enter__(self):
        return self.ptr

    def __exit__(self, *exc):
        if self._keep is None:
            self._sim.device_free(self.ptr)


def _depth(depth):
    return -1 if depth is None else int(depth)


def _is_tensor(a):
    return not isinstance(a, np.ndarray) and hasattr(a, "data_ptr")


def mat4_to_struct(m):
    """Row-major 4x4 math matrix -> mat4 (rows[]). The reference host stores glm::transpose(M)."""
    m = np.asarray(m, dtype=np.float32).reshape(4, 4)
    out = Mat4()
    for r in range(4):
        out.rows[r] = Float4(*[float(v) for v in m[r]])
    return out


class SimLOD:
    """One octree builder + rasteriser instance on one GPU (the reference is one per process)."""

    def __init__(self, width=1920, height=1080, device=0, momentary_bytes=0, nodes_bytes=0, renderbuffer_bytes=0,
                 persistent_bytes=0, construct_blocks_per_sm=0, render_blocks_per_sm=0):
        self._lib = load_library()
        self._ctx = C.c_void_p()
        cfg = Config(device, width, height, momentary_bytes, nodes_bytes, renderbuffer_bytes, persistent_bytes,
                     construct_blocks_per_sm, render_blocks_per_sm)
        self._check(self._lib.simlod_create(C.byref(cfg), C.byref(self._ctx)))
        self.width, self.height, self.device = width, height, device
        self.uniforms = Uniforms()
        self._lib.simlod_get_uniforms(self._ctx, C.byref(self.uniforms))
        # settings defaults of the reference GUI (main.cpp:123-139), except HQS: the path named by
        # the benchmark is the 64-bit atomicMin splat
        self.uniforms.showPoints = 1
        self.uniforms.doUpdateVisibility = 1
        self.uniforms.LOD = 0.2
        self.uniforms.minNodeSize = 64.0
        self.uniforms.pointSize = 1
        self.uniforms.useHighQualityShading = 0
        self.uniforms.enableEDL = 1
        self.uniforms.edlStrength = 0.8
        self.uniforms.fovy_rad = 3.1415 * 60.0 / 180.0
        ident = np.eye(4, dtype=np.float32)
        for name in ("world", "view", "proj", "transform", "transform_updateBound", "transformInv_updateBound"):
            setattr(self.uniforms, name, mat4_to_struct(ident))
        self._push_uniforms()

    # -- plumbing -------------------------------------------------------------------------------
    def _check(self, rc):
        if rc != 0:
            raise SimlodError(rc, self._lib.simlod_last_error().decode())

    def _call(self, fn, info, *args):
        """fn(ctx, *args, &info, &kernel_ms), raising SimlodError on failure. Returns (info, kernel ms)."""
        ms = C.c_float(0)
        self._check(fn(self._ctx, *args, C.byref(info), C.byref(ms)))
        return info, ms.value

    def _push_uniforms(self):
        self._check(self._lib.simlod_set_uniforms(self._ctx, C.byref(self.uniforms)))
        self._lib.simlod_get_uniforms(self._ctx, C.byref(self.uniforms))

    def close(self):
        if self._ctx:
            self._lib.simlod_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- getUniforms (main.cpp:283-331) -----------------------------------------------------------
    def set_box(self, box_min, box_max):
        """Bounding box of the point set; the host passes boxMin = 0 and boxMax = size (main.cpp:312-313)."""
        for i in range(3):
            self.uniforms.boxMin[i] = float(box_min[i])
            self.uniforms.boxMax[i] = float(box_max[i])
        self._push_uniforms()

    def set_camera(self, view, proj, update_visibility=True):
        """view/proj: row-major 4x4 math matrices (float64 ok). transform = proj * view * world(identity)."""
        view32 = np.asarray(view, dtype=np.float32).reshape(4, 4)
        proj32 = np.asarray(proj, dtype=np.float32).reshape(4, 4)
        wvp = (proj32 @ view32).astype(np.float32)
        self.uniforms.world = mat4_to_struct(np.eye(4, dtype=np.float32))
        self.uniforms.view = mat4_to_struct(view32)
        self.uniforms.proj = mat4_to_struct(proj32)
        self.uniforms.transform = mat4_to_struct(wvp)
        if update_visibility:                      # settings.doUpdateVisibility (main.cpp:300-306)
            self.uniforms.transform_updateBound = mat4_to_struct(wvp)
            self.uniforms.transformInv_updateBound = mat4_to_struct(np.linalg.inv(wvp.astype(np.float64)).astype(np.float32))
        self._push_uniforms()

    def set_settings(self, **kw):
        for k, v in kw.items():
            if not hasattr(self.uniforms, k):
                raise AttributeError(k)
            setattr(self.uniforms, k, v)
        self._push_uniforms()

    def uniforms_bytes(self):
        return bytes(bytearray(self.uniforms))

    # -- launch surface ---------------------------------------------------------------------------
    def use_module(self, program, cubin_path):
        self._check(self._lib.simlod_use_module(self._ctx, program, cubin_path.encode() if cubin_path else None))

    def reset(self, grid=None):
        """resetCUDA. grid=(blocks, threads) picks the reset kernel's launch shape; (1, 1) is the reference's."""
        if grid is None:
            self._check(self._lib.simlod_reset(self._ctx))
        else:
            self._check(self._lib.simlod_reset_with_grid(self._ctx, int(grid[0]), int(grid[1])))

    def upload_batch(self, points):
        pts = _as_points(points)
        self._check(self._lib.simlod_upload_batch(self._ctx, pts.ctypes.data, pts.shape[0]))

    def upload_batch_device(self, device_ptr, count):
        self._check(self._lib.simlod_upload_batch_device(self._ctx, int(device_ptr), int(count)))

    @staticmethod
    def las_layout(bytes_per_point, fmt, scale, offset, translation=(0.0, 0.0, 0.0)):
        return LasLayout(bytes_per_point, fmt, (C.c_double * 3)(*scale), (C.c_double * 3)(*offset), (C.c_double * 3)(*translation))

    def upload_batch_las(self, records, count, layout):
        """Upload `count` raw LAS point records (uint8 array) and decode them on the device into the next ring slot."""
        rec = np.ascontiguousarray(records, dtype=np.uint8)
        assert rec.nbytes >= count * layout.bytes_per_point
        self._check(self._lib.simlod_upload_batch_las(self._ctx, rec.ctypes.data, int(count), C.byref(layout)))

    def upload_batch_las_device(self, device_ptr, count, layout):
        self._check(self._lib.simlod_upload_batch_las_device(self._ctx, int(device_ptr), int(count), C.byref(layout)))

    def ring_slot(self, slot, count):
        """Read back `count` points of ring slot `slot` (tests)."""
        b = self.buffers()
        return self.memcpy_dtoh(b.ring + slot * MAX_BATCH_SIZE * 16, count * 16).view(POINT_DTYPE)

    def update_octree(self):
        ms = C.c_float(0)
        self._check(self._lib.simlod_update_octree(self._ctx, C.byref(ms)))
        return ms.value

    def insert(self, points):
        """Stream a host point set through the ring in 1 M-point batches (uploads overlap the update
        launches). Returns (summed kernel ms, total device ms)."""
        pts = _as_points(points)
        return self.insert_host_ptr(pts.ctypes.data, pts.shape[0])

    def insert_host_ptr(self, host_ptr, count):
        kms, tms = C.c_float(0), C.c_float(0)
        self._check(self._lib.simlod_insert(self._ctx, int(host_ptr), int(count), C.byref(kms), C.byref(tms)))
        return kms.value, tms.value

    def insert_device(self, device_ptr, count):
        kms, tms = C.c_float(0), C.c_float(0)
        self._check(self._lib.simlod_insert_device(self._ctx, int(device_ptr), int(count), C.byref(kms), C.byref(tms)))
        return kms.value, tms.value

    def insert_simlod_file(self, path, loader_threads=16, direct=False):
        """reload() of the reference for one .simlod file: reset, stream the file through pinned slots with
        `loader_threads` reader threads, insert. direct=True reads unbuffered (O_DIRECT), for files that are not in
        the page cache. Returns (num_points, summed kernel ms, total device ms)."""
        n, kms, tms = C.c_uint64(), C.c_float(), C.c_float()
        self._check(self._lib.simlod_insert_simlod_file_ex(self._ctx, path.encode(), int(loader_threads), 1 if direct else 0, C.byref(n), C.byref(kms), C.byref(tms)))
        self._lib.simlod_get_uniforms(self._ctx, C.byref(self.uniforms))
        return n.value, kms.value, tms.value

    def insert_files(self, paths, loader_threads=16, direct=False):
        """reload() of the reference for a list of .las / .simlod files (simlod_insert_files): validate every file (on
        error nothing changes), set the union box, reset, and stream the files' 1 M-point batches in list order, LAS
        records decoded on the device. direct=True reads unbuffered (O_DIRECT). Returns (num_points, summed kernel ms,
        total device ms)."""
        paths = [os.fsencode(p) for p in paths]
        arr = (C.c_char_p * max(1, len(paths)))(*paths)
        n, kms, tms = C.c_uint64(), C.c_float(), C.c_float()
        rc = self._lib.simlod_insert_files(self._ctx, arr, len(paths), int(loader_threads), 1 if direct else 0, C.byref(n), C.byref(kms), C.byref(tms))
        self._lib.simlod_get_uniforms(self._ctx, C.byref(self.uniforms))
        self._check(rc)
        return n.value, kms.value, tms.value

    def save_octree(self, path):
        """Save the octree, as the last completed update left it, to an octree file (simlod_save_octree): the full
        export's records and samples (np.memmap-able at the header's offsets), the nodes' counters, the box and the batch
        counters. Writes nothing into the context. Returns (ExportInfo, kernel ms)."""
        return self._call(self._lib.simlod_save_octree, ExportInfo(), os.fsencode(path))

    def load_octree(self, path, loader_threads=16):
        """Replace the octree by an octree file's (simlod_load_octree): render it, export it or insert further batches,
        which continue as they would have in the context that saved it. Sets the box of the uniforms; the camera and
        settings stay. Returns (ExportInfo, kernel ms)."""
        info, ms = ExportInfo(), C.c_float(0)
        rc = self._lib.simlod_load_octree(self._ctx, os.fsencode(path), int(loader_threads), C.byref(info), C.byref(ms))
        self._lib.simlod_get_uniforms(self._ctx, C.byref(self.uniforms))
        self._check(rc)
        return info, ms.value

    def write_las_into(self, path, params, samples_ptr, num_samples, depth):
        """simlod_write_las with SimlodLasWriteParams: samples_ptr 0 for the octree source (depth None or < 0: the
        inserted points), else num_samples 16-byte samples at a 16-byte aligned device address. Returns (LasWriteInfo,
        kernel ms); on SimlodError the info is the exception's `.info` (first_invalid names an invalid sample)."""
        info, ms = LasWriteInfo(), C.c_float(0)
        rc = self._lib.simlod_write_las(self._ctx, os.fsencode(path), C.byref(params), int(samples_ptr), int(num_samples), _depth(depth),
                                        C.byref(info), C.byref(ms))
        if rc != 0:
            err = SimlodError(rc, self._lib.simlod_last_error().decode())
            err.info = info
            raise err
        return info, ms.value

    def write_las(self, path, samples=None, depth=None, scale=0.001, offset=None, translation=(0.0, 0.0, 0.0), writer_threads=8):
        """Write samples to a LAS 1.2 file (point format 2), quantised and encoded on the GPU (simlod_write_las).

        Record i of the file is sample i of the source: of `samples`, or with samples=None of
        export_octree(depth).samples for the octree as the last completed update left it (depth=None: the inserted
        points, export_octree(20), those on the cube's max face included). `samples`: a CUDA float32 (N, 4) tensor (x, y,
        z, colour bits; used in place when contiguous and 16-byte aligned), or a numpy POINT_DTYPE or (N, 4) float32
        array (copied to the device) -- the layout export_*, query_region and the queries' samples=True return.
        Per axis, in IEEE double: q = rint(((double(p) + translation) - offset) / scale), half to even, with offset
        defaulting to translation, so a reader sees x = q * scale + offset near p + translation. `scale` is a scalar or
        a 3-tuple. A non-finite coordinate or a q outside int32 refuses the call, naming the first such sample in
        SimlodError.info.first_invalid; a failed call leaves no file and an existing file at `path` as it was.
        Colours become R, G, B = 257 * colour byte (alpha dropped). Returns the LasWriteInfo."""
        params = las_write_params(scale, offset, translation, writer_threads)
        if samples is None:
            return self.write_las_into(path, params, 0, 0, depth)[0]
        if _is_tensor(samples):
            import torch
            if not samples.is_cuda or samples.dtype != torch.float32 or samples.ndim != 2 or samples.shape[1] != 4:
                raise ValueError("samples must be a CUDA float32 (N, 4) tensor, or a POINT_DTYPE or (N, 4) float32 array")
            a = samples if samples.shape[0] and samples.data_ptr() else np.zeros((0, 4), dtype=np.float32)
        else:
            a = np.asarray(samples)
            if a.dtype == POINT_DTYPE:
                a = a.reshape(-1).view(np.float32).reshape(-1, 4)
            if a.dtype != np.float32 or a.ndim != 2 or a.shape[1] != 4:
                raise ValueError("samples must be a CUDA float32 (N, 4) tensor, or a POINT_DTYPE or (N, 4) float32 array")
            a = np.ascontiguousarray(a)
        with _DeviceInput(self, a) as ptr:                   # an empty array still gets an address: 0 is the octree
            return self.write_las_into(path, params, ptr, a.shape[0], depth)[0]

    def insert_batches(self, batches):
        """Insert explicit batches (each <= 1 M points), each followed by update launches until the
        device has consumed it (one batch per addBatch, as when the loader is slower than the GPU).
        Returns the summed kernel ms. Raises SimlodError(SIMLOD_ERR_CAPACITY = -5) as soon as the builder refuses a batch
        because the persistent heap is almost full, as simlod_insert* do."""
        total = 0.0
        done = self.stats().batchletIndex
        for b in batches:
            self.upload_batch(b)
            done += 1
            while True:
                total += self.update_octree()
                s = self.stats()
                if s.memCapacityReached:
                    raise SimlodError(-5, "persistent heap almost full after %d points" % s.numPointsProcessed)
                if s.batchletIndex >= done:
                    break
        return total

    def set_clip(self, regions, mode="inside"):
        """Clip what render() and pick() draw (simlod_set_clip): with mode="inside" only the samples of the LOD cut inside
        `regions`, with mode="outside" only those outside. `regions` is one Region (Region.box / sphere / planes) or a
        list of up to 4, whose union is clipped by; a sample is inside by the region query's float32 predicate on its
        stored x, y, z. None clears the clip. The cut, the visibility flags, stats() and export_view() do not change, so
        pick indices stay indices into export_view().samples. The clip stays until it is set again. A malformed region,
        an empty list or more than 4 regions raise SimlodError(-2) and leave the previous clip in place."""
        clip = SimlodClip()
        if regions is not None:
            modes = {"inside": CLIP_INSIDE, "outside": CLIP_OUTSIDE}
            if mode not in modes:
                raise ValueError("mode must be 'inside' or 'outside', not %r" % (mode,))
            regions = [regions] if isinstance(regions, SimlodRegion) else list(regions)
            clip.mode, clip.num_regions = modes[mode], len(regions)
            for k, r in enumerate(regions[:CLIP_MAX_REGIONS]):
                clip.regions[k] = r
        self._check(self._lib.simlod_set_clip(self._ctx, C.byref(clip)))

    def render(self):
        ms = C.c_float(0)
        self._check(self._lib.simlod_render(self._ctx, C.byref(ms)))
        return ms.value

    def stats(self):
        s = Stats()
        self._check(self._lib.simlod_get_stats(self._ctx, C.byref(s)))
        return s

    def framebuffer(self):
        out = np.empty((self.height, self.width), dtype=np.uint64)
        self._check(self._lib.simlod_read_framebuffer(self._ctx, out.ctypes.data))
        return out

    def surface(self):
        out = np.empty((self.height, self.width), dtype=np.uint32)
        self._check(self._lib.simlod_read_surface(self._ctx, out.ctypes.data))
        return out

    def buffers(self):
        b = Buffers()
        self._check(self._lib.simlod_get_buffers(self._ctx, C.byref(b)))
        return b

    def memcpy_dtoh(self, device_ptr, nbytes):
        out = np.empty(int(nbytes), dtype=np.uint8)
        if nbytes:
            self._check(self._lib.simlod_memcpy_dtoh(self._ctx, out.ctypes.data, int(device_ptr), int(nbytes)))
        return out

    def memcpy_htod(self, device_ptr, array):
        a = np.ascontiguousarray(array)
        self._check(self._lib.simlod_memcpy_htod(self._ctx, int(device_ptr), a.ctypes.data, a.nbytes))

    def download_octree(self):
        """Raw octree image for canonicalisation: (nodes bytes, heap bytes, nodes device address, heap device address)."""
        s = self.stats()
        b = self.buffers()
        nodes = self.memcpy_dtoh(b.nodes, s.numNodes * NODE_BYTES)
        heap_used = int(self.memcpy_dtoh(b.persistent + 8, 8).view(np.uint64)[0])
        heap = self.memcpy_dtoh(b.persistent, heap_used)
        return nodes, heap, int(b.nodes), int(b.persistent)

    def export_octree_into(self, depth, dst_nodes, node_capacity, dst_samples, sample_capacity):
        """simlod_export_octree into caller-owned device memory (depth None or < 0: full export; all zero: size query).
        Returns (ExportInfo, kernel ms)."""
        return self._call(self._lib.simlod_export_octree, ExportInfo(), _depth(depth), int(dst_nodes), int(node_capacity),
                          int(dst_samples), int(sample_capacity))

    def export_octree(self, depth=None, device="cuda"):
        """The octree as flat arrays (simlod_export_octree): depth=None exports every node with its points and voxels, an
        integer depth the cut at that level (the voxels of the inner nodes at `depth`, the points of the leaves above).
        Returns an OctreeExport: `nodes` (numpy EXPORT_NODE_DTYPE), `samples` and `info` (ExportInfo). With device="cuda"
        the samples stay in device memory as a float32 torch tensor of shape (N, 4) (x, y, z, colour bits:
        `.view(torch.int32)[:, 3]` is the colour); with device="cpu" they are a numpy POINT_DTYPE array."""
        return self._export(lambda *dst: self.export_octree_into(depth, *dst), device)

    def export_view_into(self, dst_nodes, node_capacity, dst_samples, sample_capacity):
        """simlod_export_view into caller-owned device memory (all zero: size query). Returns (ExportInfo, kernel ms)."""
        return self._call(self._lib.simlod_export_view, ExportInfo(), int(dst_nodes), int(node_capacity), int(dst_samples),
                          int(sample_capacity))

    def export_view(self, device="cuda"):
        """The LOD cut render() draws for the current camera and settings, as flat arrays (simlod_export_view): the drawn
        nodes flagged EXPORT_SAMPLED with their points and voxels, and the records that link them to the root. Writes no
        visibility flags. Returns an OctreeExport, with `samples` on `device` as for export_octree."""
        return self._export(self.export_view_into, device)

    def _export(self, into, device):
        """Size query, then the export into arrays of that size: into(dst_nodes, node_capacity, dst_samples,
        sample_capacity) -> (ExportInfo, ms)."""
        info, _ = into(0, 0, 0, 0)
        n, m = info.num_nodes, info.num_samples
        with _Results(self, device, (((n,), EXPORT_NODE_DTYPE), ((m,), POINT_DTYPE))) as r:
            info, _ = into(r.ptrs[0], n, r.ptrs[1], m)
            return OctreeExport(*r.results(), info)

    def query_region_into(self, region, depth, dst_samples, sample_capacity):
        """simlod_query_region into caller-owned device memory (depth None or < 0: the inserted points; dst_samples 0:
        size query). Returns (SimlodQueryInfo, kernel ms)."""
        return self._call(self._lib.simlod_query_region, SimlodQueryInfo(), C.byref(region), _depth(depth), int(dst_samples),
                          int(sample_capacity))

    def query_region(self, region, depth=None, device="cuda"):
        """The samples inside `region` (Region.box / sphere / planes), filtered on the GPU (simlod_query_region): with
        depth=None the inserted points, with an integer depth the samples of the cut at that level (as export_octree), so
        that a coarse preview costs a coarse amount of work. Points outside the half-open octree cube (in practice those
        exactly on its max face) are never returned. The order is deterministic. Returns (samples, SimlodQueryInfo):
        with device="cuda" a float32 torch tensor of shape (N, 4) in device memory (x, y, z, colour bits), with
        device="cpu" a numpy POINT_DTYPE array."""
        info, _ = self.query_region_into(region, depth, 0, 0)
        m = info.num_samples
        with _Results(self, device, (((m,), POINT_DTYPE),)) as r:
            if m:
                info, _ = self.query_region_into(region, depth, r.ptrs[0], m)
            return r.results()[0], info

    def pick_into(self, pixels, dst_index, dst_samples):
        """simlod_pick into caller-owned device memory: pixels None for the whole frame, else an (N, 2) array of (x, y);
        dst_index (int64) and dst_samples (16-byte samples, 0 for none) both 0: info only. Returns (SimlodPickInfo,
        kernel ms)."""
        if pixels is None:
            ptr, n = None, 0
        else:
            a = np.asarray(pixels)
            if a.ndim != 2 or a.shape[1] != 2 or (a.size and a.dtype.kind not in "iu"):
                raise ValueError("pixels must be an (N, 2) integer array of (x, y)")
            a = a.astype(np.int64)
            # negative or huge coordinates become ones the library refuses as outside the frame
            a = np.ascontiguousarray(np.where((a < 0) | (a > 0xFFFFFFFF), 0xFFFFFFFF, a).astype(np.uint32))
            n = a.shape[0]
            keep = a if n else np.zeros(2, dtype=np.uint32)        # an empty list is still a list (and is refused)
            ptr = keep.ctypes.data_as(C.POINTER(C.c_uint32))
        return self._call(self._lib.simlod_pick, SimlodPickInfo(), ptr, n, int(dst_index), int(dst_samples))

    def pick(self, pixels=None, device="cuda", samples=False):
        """The sample under each pixel of the frame render() draws for the current uniforms (simlod_pick): an index into
        export_view().samples, -1 where the frame shows no sample. pixels=None picks the whole frame, an (H, W) int64
        result; an (N, 2) array of (x, y) with x < width and y < height picks those pixels, an (N,) result. With
        samples=True the picked samples are returned too, (H, W, 4) or (N, 4) float32 in the export's layout (x, y, z,
        colour bits), zeros where the index is -1. device="cuda": torch tensors in device memory; device="cpu": numpy
        arrays (the samples as POINT_DTYPE). Returns (index, info) or, with samples=True, (index, samples, info)."""
        shape = (self.height, self.width) if pixels is None else (len(np.asarray(pixels)),)
        with _Results(self, device, ((shape, I8), (shape, POINT_DTYPE) if samples else None)) as r:
            info, _ = self.pick_into(pixels, *r.ptrs)
            return r.results() + (info,)

    def query_nearest_into(self, queries_ptr, n, k, depth, max_radius, dst_index, dst_dist2, dst_samples):
        """simlod_query_nearest on caller-owned device memory: n 16-byte query records at queries_ptr, destinations
        [n][k] int64 / float32 / 16-byte samples, each 0 for not written (depth None or < 0: the inserted points;
        max_radius None: no limit). Returns (SimlodNearestInfo, kernel ms)."""
        r = float("inf") if max_radius is None else float(max_radius)
        return self._call(self._lib.simlod_query_nearest, SimlodNearestInfo(), int(queries_ptr), int(n), int(k), _depth(depth), r,
                          int(dst_index), int(dst_dist2), int(dst_samples))

    def query_nearest(self, queries, k=8, depth=None, max_radius=None, device="cuda", samples=False):
        """The k nearest samples of each query position (simlod_query_nearest), exact: with depth=None among the
        inserted points (those on the cube's max face excepted, as query_region), with an integer depth among the
        samples of export_octree(depth). Samples are ordered by squared distance in float32, ties by index, and only
        those within max_radius count. `queries`: an (N, 3) or (N, 4) array (the 4th column is ignored), numpy or a CUDA
        tensor, or POINT_DTYPE samples. Returns (index, dist2, info) or, with samples=True, (index, dist2, samples, info):
        (N, k) int64 indices into export_octree(depth).samples, -1 in an empty slot; (N, k) float32 squared distances,
        +inf in an empty slot; (N, k, 4) float32 samples in the export's layout, zeros in an empty slot. device="cuda":
        torch tensors in device memory; device="cpu": numpy arrays (the samples as POINT_DTYPE)."""
        with self._device_queries(queries) as (qptr, n):
            return self._nearest(qptr, n, k, depth, max_radius, device, samples)

    @contextlib.contextmanager
    def _device_queries(self, queries):
        """The query records query_nearest and query_radius take, as 16-byte records (x, y, z, ignored word) at a device
        address: yields (address, count). `queries`: an (N, 3) or (N, 4) array (the 4th column is ignored), numpy or a
        CUDA tensor, or POINT_DTYPE samples. A contiguous float32 (N, 4) CUDA tensor at a 16-byte aligned address is
        passed as it is; anything else is copied, into memory freed when the block ends."""
        if isinstance(queries, np.ndarray) and queries.dtype == POINT_DTYPE:
            queries = queries.view(np.float32).reshape(-1, 4)
        if _is_tensor(queries):
            import torch
            if not queries.is_cuda or queries.ndim != 2 or queries.shape[1] not in (3, 4):
                raise ValueError("queries must be an (N, 3) or (N, 4) CUDA tensor or numpy array")
            q = queries.detach().to(torch.float32)
            if q.shape[1] == 3:
                q = torch.cat([q, q.new_zeros((q.shape[0], 1))], dim=1)
        else:
            a = np.asarray(queries)
            if a.ndim != 2 or a.shape[1] not in (3, 4):
                raise ValueError("queries must be an (N, 3) or (N, 4) CUDA tensor or numpy array")
            q = np.zeros((a.shape[0], 4), dtype=np.float32)
            q[:, :3] = a[:, :3]
        with _DeviceInput(self, q) as ptr:
            yield ptr, q.shape[0]

    def _nearest(self, qptr, n, k, depth, max_radius, device, samples):
        with _Results(self, device, (((n, k), I8), ((n, k), F4), ((n, k), POINT_DTYPE) if samples else None)) as r:
            info, _ = self.query_nearest_into(qptr, n, k, depth, max_radius, *r.ptrs)
            return r.results() + (info,)

    def query_radius_into(self, queries_ptr, n, radius, depth, dst_offsets, dst_index, dst_dist2, dst_samples, capacity):
        """simlod_query_radius on caller-owned device memory: n 16-byte query records at queries_ptr; dst_offsets int64
        [n + 1]; dst_index / dst_dist2 / dst_samples int64 / float32 / 16-byte samples with `capacity` neighbour slots
        each, 0 for not written (all three 0: size query, which fills the offsets when dst_offsets is not 0; depth None or
        < 0: the inserted points). Returns (SimlodRadiusInfo, kernel ms)."""
        return self._call(self._lib.simlod_query_radius, SimlodRadiusInfo(), int(queries_ptr), int(n), float(radius), _depth(depth),
                          int(dst_offsets), int(dst_index), int(dst_dist2), int(dst_samples), int(capacity))

    def query_radius(self, queries, radius, depth=None, device="cuda", samples=False):
        """Every sample within `radius` of each query position (simlod_query_radius), exact: with depth=None among the
        inserted points (those on the cube's max face excepted, as query_region), with an integer depth among the
        samples of export_octree(depth). A sample is a neighbour when its squared distance in float32, the k-nearest
        query's key, is <= radius * radius. `queries` as query_nearest takes them. The result is in CSR form: query q's
        neighbours are [offsets[q], offsets[q + 1]) of index (int64 indices into export_octree(depth).samples), dist2
        (float32) and, with samples=True, samples ((M, 4) float32 in the export's layout). Within a query the records
        come in Z-order and each record's samples in the export's order (not sorted by distance or index). A query with
        a non-finite coordinate has no neighbours and counts in info.invalid_queries. One size query, then the full
        call. Returns (offsets, index, dist2, info) or, with samples=True, (offsets, index, dist2, samples, info).
        device="cuda": torch tensors in device memory; device="cpu": numpy arrays (the samples as POINT_DTYPE)."""
        with self._device_queries(queries) as (qptr, n):
            info, _ = self.query_radius_into(qptr, n, radius, depth, 0, 0, 0, 0, 0)
            m = info.num_found
            with _Results(self, device, (((n + 1,), I8), ((m,), I8), ((m,), F4), ((m,), POINT_DTYPE) if samples else None), keep=True) as r:
                info, _ = self.query_radius_into(qptr, n, radius, depth, *r.ptrs, m)
                return r.results() + (info,)

    def query_ray_into(self, rays_ptr, n, radius, depth, dst_index, dst_t, dst_h2, dst_samples):
        """simlod_query_ray on caller-owned device memory: n 32-byte ray records (ox, oy, oz, tmin, dx, dy, dz, tmax) at
        rays_ptr, destinations [n] int64 / float32 / float32 / 16-byte samples, each 0 for not written (depth None or < 0:
        the inserted points). Returns (SimlodRayInfo, kernel ms)."""
        return self._call(self._lib.simlod_query_ray, SimlodRayInfo(), int(rays_ptr), int(n), float(radius), _depth(depth),
                          int(dst_index), int(dst_t), int(dst_h2), int(dst_samples))

    def query_ray(self, origins, directions, radius, tmin=0.0, tmax=None, depth=None, device="cuda", samples=False):
        """The first stored sample along each ray (simlod_query_ray), exact: among the samples within `radius` of the ray
        o + t u (u the direction normalised by the library) with tmin <= t <= tmax, the one with the least t, ties by
        index. With depth=None among the inserted points (those on the cube's max face excepted, as query_region), with
        an integer depth among the samples of export_octree(depth). `origins`, `directions`: (N, 3) arrays, numpy or CUDA
        tensors; `tmin`, `tmax`: scalars or (N,) arrays (tmax None: +inf). A ray with a non-finite or zero direction, a
        non-finite origin or a bad [tmin, tmax] gets an empty result and counts in info.invalid_rays. Returns
        (index, t, h2, info) or, with samples=True, (index, t, h2, samples, info): (N,) int64 indices into
        export_octree(depth).samples, -1 for no hit; (N,) float32 t, +inf for no hit; (N,) float32 squared distances
        from the ray, +inf for no hit; (N, 4) float32 samples in the export's layout, zeros for no hit. device="cuda":
        torch tensors in device memory; device="cpu": numpy arrays (the samples as POINT_DTYPE)."""
        if _is_tensor(origins):
            import torch
            o = origins.detach()
            d = directions.detach() if hasattr(directions, "data_ptr") else torch.as_tensor(np.asarray(directions), device=o.device)
            if not o.is_cuda or o.ndim != 2 or o.shape[1] != 3 or tuple(d.shape) != tuple(o.shape):
                raise ValueError("origins and directions must be (N, 3) CUDA tensors or numpy arrays of one shape")
            n = o.shape[0]
            r = torch.empty((n, 8), dtype=torch.float32, device=o.device)
            r[:, 0:3] = o.to(torch.float32)
            r[:, 4:7] = d.to(device=o.device, dtype=torch.float32)
            for col, v, default in ((3, tmin, 0.0), (7, tmax, float("inf"))):
                v = default if v is None else v
                r[:, col] = v.to(device=o.device, dtype=torch.float32) if hasattr(v, "data_ptr") else \
                    torch.as_tensor(np.broadcast_to(np.asarray(v, dtype=np.float32), (n,)).copy(), device=o.device)
        else:
            o, d = np.asarray(origins), np.asarray(directions)
            if o.ndim != 2 or o.shape[1] != 3 or d.shape != o.shape:
                raise ValueError("origins and directions must be (N, 3) CUDA tensors or numpy arrays of one shape")
            n = o.shape[0]
            r = np.empty((n, 8), dtype=np.float32)
            r[:, 0:3], r[:, 4:7] = o, d
            r[:, 3] = np.broadcast_to(np.asarray(0.0 if tmin is None else tmin, dtype=np.float32), (n,))
            r[:, 7] = np.broadcast_to(np.asarray(np.inf if tmax is None else tmax, dtype=np.float32), (n,))
        with _DeviceInput(self, r) as rptr, _Results(self, device, (((n,), I8), ((n,), F4), ((n,), F4), ((n,), POINT_DTYPE) if samples else None)) as out:
            info, _ = self.query_ray_into(rptr, n, radius, depth, *out.ptrs)
            return out.results() + (info,)

    def query_heightmap_into(self, grid, depth, dst_count, dst_z_min, dst_z_max, dst_z_mean, dst_top, dst_samples):
        """simlod_query_heightmap on caller-owned device memory: `grid` a SimlodHeightmap, destinations [ny][nx] int64 /
        float32 / float32 / float32 / int64 / 16-byte samples, each 0 for not written (depth None or < 0: the inserted
        points). Returns (SimlodHeightmapInfo, kernel ms)."""
        return self._call(self._lib.simlod_query_heightmap, SimlodHeightmapInfo(), C.byref(grid), _depth(depth), int(dst_count),
                          int(dst_z_min), int(dst_z_max), int(dst_z_mean), int(dst_top), int(dst_samples))

    def query_heightmap(self, origin, cell, shape, depth=None, device="cuda", samples=False):
        """A height map of the stored samples (simlod_query_heightmap), exact: per cell of the grid of square cells of
        edge `cell` with cell (0, 0) at `origin` (x, y), the samples whose u = (x - ox) / cell and v = (y - oy) / cell
        (float32, IEEE division) satisfy u >= 0, v >= 0, trunc(u) < nx and trunc(v) < ny fall in cell (trunc(u), trunc(v)).
        With depth=None the inserted points (those on the cube's max face excepted, as query_region), with an integer
        depth the samples of export_octree(depth). `shape` is (ny, nx), at most 2^27 cells (tile larger rasters); row j,
        column i is cell (i, j), rows in +y order. Returns (count, z_min, z_max, z_mean, top, info) or, with
        samples=True, (count, z_min, z_max, z_mean, top, samples, info): (ny, nx) int64 counts; float32 lowest, highest
        and mean z, NaN for an empty cell (z ordered by its sign-aware bits, -0 below +0; the mean is that of z
        quantised to 2^-30 of the cube edge, byte-deterministic); int64 indices into export_octree(depth).samples of the
        highest sample, equal z to the smallest index, -1 for an empty cell; (ny, nx, 4) float32 samples in the export's
        layout, zeros for an empty cell. device="cuda": torch tensors in device memory; device="cpu": numpy arrays (the
        samples as POINT_DTYPE)."""
        ny, nx = (int(v) for v in shape)
        if ny < 0 or nx < 0 or ny > 0xFFFFFFFF or nx > 0xFFFFFFFF:
            raise ValueError("shape must be (ny, nx) with 0 <= nx, ny < 2^32")
        grid = SimlodHeightmap(cell=float(cell), nx=nx, ny=ny)
        grid.origin[:] = [float(v) for v in origin]
        s = (ny, nx)
        with _Results(self, device, ((s, I8), (s, F4), (s, F4), (s, F4), (s, I8), (s, POINT_DTYPE) if samples else None)) as r:
            info, _ = self.query_heightmap_into(grid, depth, *r.ptrs)
            return r.results() + (info,)

    def host_alloc(self, nbytes):
        p = C.c_void_p()
        self._check(self._lib.simlod_host_alloc(self._ctx, int(nbytes), C.byref(p)))
        return p.value

    def host_free(self, ptr):
        self._check(self._lib.simlod_host_free(self._ctx, C.c_void_p(ptr)))

    def device_alloc(self, nbytes):
        p = C.c_uint64()
        self._check(self._lib.simlod_device_alloc(self._ctx, int(nbytes), C.byref(p)))
        return p.value

    def device_free(self, ptr):
        self._check(self._lib.simlod_device_free(self._ctx, int(ptr)))

    def launch_info(self):
        n, cb, rb, sms = C.c_uint64(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._check(self._lib.simlod_get_launch_info(self._ctx, C.byref(n), C.byref(cb), C.byref(rb), C.byref(sms)))
        return {"launches": n.value, "construct_blocks": cb.value, "render_blocks": rb.value, "num_sms": sms.value}

    def numa_node(self):
        n = C.c_int(-1)
        self._check(self._lib.simlod_get_numa_node(self._ctx, C.byref(n)))
        return n.value

    def device_rcp(self, x):
        out = C.c_float()
        self._check(self._lib.simlod_device_rcp(self._ctx, float(x), C.byref(out)))
        return np.float32(out.value)

    GEN_UNIFORM, GEN_TERRAIN, GEN_SHELL = 0, 1, 2

    def generate(self, kind, device_ptr, n_total, first, count, seed, size=0.0):
        """Points [first, first+count) of a synthetic n_total-point stream (data.py generators restated on the device)."""
        self._check(self._lib.simlod_generate(self._ctx, int(kind), int(n_total), int(first), int(count), int(seed), float(size), int(device_ptr)))

    def synchronize(self):
        self._check(self._lib.simlod_synchronize(self._ctx))

    def flush_l2(self):
        self._check(self._lib.simlod_flush_l2(self._ctx))

    # ---- spatial exchange (one octree over several GPUs) ----
    @staticmethod
    def partition_plan(level, owners, num_ranks):
        owners = np.asarray(owners, dtype=np.uint8)
        if owners.shape != (8 ** level,):
            raise ValueError("need %d owners for level %d" % (8 ** level, level))
        plan = PartitionPlan(level, num_ranks)
        C.memmove(plan.owner, owners.ctypes.data, owners.size)
        return plan

    def partition_count(self, device_ptr, count, plan):
        """(points per destination rank, points per level-`level` cell) of the batch at device_ptr."""
        ranks = (C.c_uint64 * plan.num_ranks)()
        cells = (C.c_uint64 * (8 ** plan.level))()
        self._check(self._lib.simlod_partition_count(self._ctx, int(device_ptr), int(count), C.byref(plan), ranks, cells))
        return np.array(ranks[:], dtype=np.uint64), np.array(cells[:], dtype=np.uint64)

    def partition_scatter(self, device_ptr, count, plan, dest_ptrs, dest_offsets, signal_ptrs=None, signal_value=0):
        ptrs = (C.c_uint64 * plan.num_ranks)(*[int(p) for p in dest_ptrs])
        offs = (C.c_uint64 * plan.num_ranks)(*[int(o) for o in dest_offsets])
        sig = (C.c_uint64 * plan.num_ranks)(*[int(p) for p in signal_ptrs]) if signal_ptrs is not None else None
        self._check(self._lib.simlod_partition_scatter(self._ctx, int(device_ptr), int(count), C.byref(plan), ptrs, offs, sig, int(signal_value)))

    def export_framebuffer(self, dst_device_ptr):
        self._check(self._lib.simlod_export_framebuffer(self._ctx, int(dst_device_ptr)))

    def peer_signal(self, signal_ptrs, value):
        sig = (C.c_uint64 * len(signal_ptrs))(*[int(p) for p in signal_ptrs])
        self._check(self._lib.simlod_peer_signal(self._ctx, sig, len(signal_ptrs), int(value)))

    def composite_framebuffers(self, fb_ptrs, rank, signal_ptrs=None, signal_value=0):
        n = len(fb_ptrs)
        fbs = (C.c_uint64 * n)(*[int(p) for p in fb_ptrs])
        sig = (C.c_uint64 * n)(*[int(p) for p in signal_ptrs]) if signal_ptrs is not None else None
        self._check(self._lib.simlod_composite_framebuffers(self._ctx, fbs, n, int(rank), sig, int(signal_value)))

    def partition_wait(self, local_flags_ptr, num_ranks, value, timeout_ms=0):
        self._check(self._lib.simlod_partition_wait(self._ctx, int(local_flags_ptr), int(num_ranks), int(value), int(timeout_ms)))
