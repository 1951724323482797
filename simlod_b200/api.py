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
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsimlod_b200.so")

POINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("color", "<u4")])

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


class PartitionPlan(C.Structure):
    """SimlodPartitionPlan: the level-`level` cells of the octree cube and the rank that owns each."""
    _fields_ = [("level", C.c_uint32), ("num_ranks", C.c_uint32), ("owner", C.c_uint8 * 512)]


class Buffers(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "nodes", "nodes_bytes", "persistent", "persistent_bytes", "momentary", "momentary_bytes",
        "renderbuffer", "renderbuffer_bytes", "ring", "ring_bytes", "stats")]


assert C.sizeof(Uniforms) == 480 and C.sizeof(Stats) == 112

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
    }
    for name, argtypes in sig.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = None if name == "simlod_destroy" else C.c_int
    _lib = lib
    return lib


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

    def insert_batches(self, batches):
        """Insert explicit batches (each <= 1 M points), each followed by update launches until the
        device has consumed it (one batch per addBatch, as when the loader is slower than the GPU).
        Returns the summed kernel ms."""
        total = 0.0
        done = self.stats().batchletIndex
        for b in batches:
            self.upload_batch(b)
            done += 1
            while True:
                total += self.update_octree()
                s = self.stats()
                if s.batchletIndex >= done or s.memCapacityReached:
                    break
        return total

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
