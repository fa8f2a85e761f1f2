"""Host-side mirror of `GaussianSplattingRasterizer` (util/gaussian_splatting_rasterizer.gd) on top of libgsr.

Same public surface as the GDScript class -- `_init(point_cloud, output_texture_size, render_texture,
camera)`, `init_gpu()`, `rasterize()`, `texture_size` setter, `update_camera_matrices() -> bool`,
`get_splat_position(Vector2i) -> Vector3`, `cleanup_gpu()`, the knobs `should_enable_heatmap`,
`render_scale`, `model_scale`, `basis_override`, `is_loaded`, `num_splats_loaded` -- so the parity tests read
like the reference's own call sites (main.gd:121-152).  Everything GPU-side goes through the C-ABI.

`render_texture` here is a `RenderTexture` holder: after `rasterize()` it exposes the device pointer of the
RGBA32F frame (the Texture2DRD's RID in the reference) and `read()` copies it to a numpy array.
"""
from __future__ import annotations

import ctypes as C
import math
import time as _time

import numpy as np

from . import _lib
from .camera import Camera3D, pack_camera_push_constants, transform_to_projection
from .compressed_ply import CompressedPlyFile
from .ply_file import PlyFile, PlyLayout, load_gaussian_splats

TILE_SIZE = 16            # rasterizer.gd:4
WORKGROUP_SIZE = 512      # rasterizer.gd:5
RADIX = 256               # rasterizer.gd:6
PARTITION_DIVISION = 8    # rasterizer.gd:7
PARTITION_SIZE = PARTITION_DIVISION * WORKGROUP_SIZE

VECTOR3_INF = np.array([np.inf, np.inf, np.inf], dtype=np.float32)


class RenderTexture:
    """Stand-in for Texture2DRD: holds the device pointer of the frame."""

    def __init__(self):
        self.device_ptr = 0
        self.size = (0, 0)
        self._owner = None

    def read(self) -> np.ndarray:
        if self._owner is None:
            raise RuntimeError("render texture is not bound to a rasterizer")
        return self._owner.read_framebuffer()


class GaussianSplattingRasterizer:
    def __init__(self, point_cloud: PlyFile, output_texture_size, render_texture: RenderTexture | None, camera: Camera3D,
                 device: int = 0, flags: int = 0, dup_capacity_factor: int = 10, clock=None, sh_bands: int | None = None,
                 antialiasing: float | None = None, depth_order: int = 0, sh_half: bool = False):
        """sh_bands: SH bands the context stores (gsr_config.sh_bands, 1..4 = degree + 1); None = the file's degree + 1, or 4 when its
        properties do not name a 3DGS layout.
        antialiasing: the 2D filter variance of anti-aliased trainings (include/gsr.h gsr_set_antialiasing; 0 = off); None = 0.1, the
        Mip-Splatting filter, when the file carries `filter_3D`, else off.  A file with `filter_3D` is loaded with its 3D filter folded
        into scale and opacity (gsr_upload_ply_filtered) whatever this value is.
        depth_order: how each tile's splats are ordered (include/gsr.h gsr_set_depth_order): 0 = the reference's 16-bit depth key, 1 = exact
        view depth (large or metric-scale scenes, depth compositing).
        sh_half: store the SH coefficients as IEEE binary16 (include/gsr.h GSR_FLAG_SH_HALF): 144 instead of 240 bytes per degree-3
        splat, each frame exactly that of the cloud with its coefficients rounded to binary16 once."""
        self.should_enable_heatmap = [False]
        self.render_scale = [1.0]
        self.model_scale = [1.0]
        self.should_terminate_thread = [False]
        self.num_splats_loaded = [0]
        self.basis_override = np.eye(3, dtype=np.float32)  # rows = basis columns x, y, z
        self.is_loaded = False
        self.loaded_callbacks = []  # signal `loaded`
        self._ctx = C.c_void_p(None)
        self._device, self._flags, self._factor = device, flags | (_lib.GSR_FLAG_SH_HALF if sh_half else 0), dup_capacity_factor
        self._compressed = isinstance(point_cloud, CompressedPlyFile)   # loaded through the device decode (upload_compressed_ply)
        if self._compressed:
            self._layout = None
        else:
            try:
                self._layout = point_cloud.layout()
            except ValueError:
                self._layout = None   # not a named 3DGS layout: the standard 62-property order, as the reference reads it
        default_bands = point_cloud.sh_degree + 1 if self._compressed else (self._layout.sh_degree + 1 if self._layout else 0)
        self._sh_bands = int(sh_bands) if sh_bands is not None else default_bands
        has_filter_3d = self._layout is not None and self._layout.filter_3d >= 0
        self._antialiasing = float(antialiasing) if antialiasing is not None else (0.1 if has_filter_3d else 0.0)
        self._depth_order = int(depth_order)
        self._cutouts = []   # gsr_cutout entries of set_cutouts, applied again by init_gpu
        self._instance_ranges = None   # (first, count) per instance of the current set_instances layout; None: no instances
        self._clock = clock or (lambda: _time.monotonic())
        self._t0 = self._clock()
        self.tile_dims = (0, 0)
        self._texture_size = (1, 1)
        self.point_cloud = point_cloud
        self.texture_size = output_texture_size
        self.render_texture = render_texture or RenderTexture()
        self.camera = camera
        self.camera_projection = None
        self.camera_transform = None
        self.camera_push_constants = None
        self._pinned = None

    # ---- texture_size setter (rasterizer.gd:26-48) ----
    @property
    def texture_size(self):
        return self._texture_size

    @texture_size.setter
    def texture_size(self, value):
        s = self.render_scale[0]
        w, h = max(1, int(value[0] * s)), max(1, int(value[1] * s))
        self._texture_size = (w, h)
        self.tile_dims = ((w + TILE_SIZE - 1) // TILE_SIZE, (h + TILE_SIZE - 1) // TILE_SIZE)
        if self._ctx:
            _lib.check(_lib.lib().gsr_resize(self._ctx, w, h), "gsr_resize")
            self._bind_texture()

    def _bind_texture(self):
        self.render_texture.device_ptr = int(_lib.lib().gsr_framebuffer_device_ptr(self._ctx) or 0)
        self.render_texture.size = self._texture_size
        self.render_texture._owner = self

    def ticks(self) -> float:
        """Time.get_ticks_msec()*1e-3 (rasterizer.gd:126, ply_file.gd:40)."""
        return self._clock() - self._t0

    # ---- init_gpu (rasterizer.gd:65-114) ----
    def init_gpu(self, load: bool = True, device_ingest: bool = False) -> None:
        """load=False creates the context only; the caller then streams splats in with `upload_splats` / `upload_ply_raw`.
        device_ingest=True runs the per-splat preprocessing of ply_file.gd:44-69 on the GPU instead of in numpy."""
        assert self.render_texture is not None, "An output Texture2DRD must be set!"
        L = _lib.lib()
        self._max_splats = max(1, self.point_cloud.size)
        cfg = _lib.GsrConfig(self._device, self._flags, self._max_splats, self._factor, self._sh_bands)
        _lib.check(L.gsr_create(C.byref(cfg), C.byref(self._ctx)), "gsr_create")
        w, h = self._texture_size
        _lib.check(L.gsr_resize(self._ctx, w, h), "gsr_resize")
        self._bind_texture()
        if self._antialiasing:
            self.set_antialiasing(self._antialiasing)
        if self._depth_order:
            self.set_depth_order(self._depth_order)
        if self._cutouts:
            self._apply_cutouts()
        self.should_terminate_thread[0] = False
        self.num_splats_loaded[0] = 0
        if not load:
            return
        if self._compressed:   # a compressed PLY is decoded on the device in one call
            self.upload_compressed_ply(self.point_cloud, 0, self.ticks())
            self._emit_loaded()
            return
        # the reference starts a loader thread (:114); here the load runs inline, chunk by chunk
        stride = max(1, self.point_cloud.size // 1000)
        if device_ingest:
            table, n, i = self.point_cloud.table, self.point_cloud.size, 0
            while i * stride < n and not self.should_terminate_thread[0]:
                lo, hi = i * stride, min(n, (i + 1) * stride)
                if self._layout is None:
                    self.upload_ply_raw(table[lo:hi], lo, self.ticks())
                else:
                    self.upload_ply(table[lo:hi], self._layout, lo, self.ticks())
                i += 1
            self._emit_loaded()
            return
        load_gaussian_splats(self.point_cloud, stride, self._upload, self.should_terminate_thread, self.num_splats_loaded,
                             self._emit_loaded, clock=self.ticks, layout=self._layout)

    def _upload(self, first: int, block60: np.ndarray) -> None:
        block60 = np.ascontiguousarray(block60, dtype=np.float32)
        _lib.check(_lib.lib().gsr_upload_splats_aos(self._ctx, block60.ctypes.data_as(C.POINTER(C.c_float)), first,
                                                    block60.shape[0]), "gsr_upload_splats_aos")

    def upload_splats(self, splat60: np.ndarray, first: int = 0) -> None:
        """Direct upload of pre-swizzled 60-float structs (used by the bench for large scenes)."""
        if not self._ctx:
            raise RuntimeError("init_gpu() first")
        self._upload(first, splat60)
        self.num_splats_loaded[0] = max(self.num_splats_loaded[0], first + splat60.shape[0])

    def upload_ply_raw(self, table: np.ndarray, first: int = 0, creation_time: float = 0.0) -> None:
        """Device-side ingest (scope row f1): raw (m, nprops) PLY vertices -> SoA planes, preprocessing on the GPU."""
        if not self._ctx:
            raise RuntimeError("init_gpu() first")
        t = np.ascontiguousarray(table, dtype=np.float32)
        _lib.check(_lib.lib().gsr_upload_ply_raw(self._ctx, t.ctypes.data_as(C.POINTER(C.c_float)), t.shape[1], first, t.shape[0],
                                                 float(creation_time)), "gsr_upload_ply_raw")
        self.num_splats_loaded[0] = max(self.num_splats_loaded[0], first + t.shape[0])

    def upload_ply(self, table: np.ndarray, layout: PlyLayout, first: int = 0, creation_time: float = 0.0) -> None:
        """Device-side ingest of PLY vertices of any SH degree and property order (include/gsr.h gsr_upload_ply); layout: PlyFile.layout().
        A layout with a `filter_3D` property goes through gsr_upload_ply_filtered (Mip-Splatting's 3D filter)."""
        if not self._ctx:
            raise RuntimeError("init_gpu() first")
        t = np.ascontiguousarray(table, dtype=np.float32)
        lay = _lib.GsrPlyLayout(layout.nprops, layout.sh_degree, layout.x, layout.f_dc, layout.f_rest, layout.opacity, layout.scale, layout.rot)
        assert t.ndim == 2 and t.shape[1] == layout.nprops, (t.shape, layout.nprops)
        ptr = t.ctypes.data_as(C.POINTER(C.c_float))
        if layout.filter_3d >= 0:
            _lib.check(_lib.lib().gsr_upload_ply_filtered(self._ctx, ptr, C.byref(lay), layout.filter_3d, first, t.shape[0], float(creation_time)),
                       "gsr_upload_ply_filtered")
        else:
            _lib.check(_lib.lib().gsr_upload_ply(self._ctx, ptr, C.byref(lay), first, t.shape[0], float(creation_time)), "gsr_upload_ply")
        self.num_splats_loaded[0] = max(self.num_splats_loaded[0], first + t.shape[0])

    def set_sh_degree(self, degree: int) -> None:
        """SH degree of the colour of the frames rendered from now on (include/gsr.h gsr_set_sh_degree): 0 .. the stored degree, -1 = the
        stored degree (the default).  A lower degree trades view-dependent colour for projection bytes."""
        _lib.check(_lib.lib().gsr_set_sh_degree(self._ctx, int(degree)), "gsr_set_sh_degree")

    def set_antialiasing(self, filter_variance: float) -> None:
        """The 2D filter of anti-aliased trainings for the frames rendered from now on (include/gsr.h gsr_set_antialiasing): 0 = off
        (the reference's +0.3 dilation), 0.3 = 3DGS --antialiasing / gsplat "antialiased", 0.1 = Mip-Splatting."""
        v = float(filter_variance)
        if self._ctx:
            _lib.check(_lib.lib().gsr_set_antialiasing(self._ctx, v), "gsr_set_antialiasing")
        self._antialiasing = v

    def set_depth_order(self, mode: int) -> None:
        """How the frames rendered from now on order each tile's splats (include/gsr.h gsr_set_depth_order): 0 = the reference's 16-bit
        depth key (ties keep splat-id order), 1 = exact view depth (ties keep splat-id order only at equal float depth)."""
        m = int(mode)
        if self._ctx:
            _lib.check(_lib.lib().gsr_set_depth_order(self._ctx, m), "gsr_set_depth_order")
        self._depth_order = m

    def set_cutouts(self, cutouts) -> None:
        """Boxes and ellipsoids that crop the cloud or cut splats away in the frames rendered from now on (include/gsr.h
        gsr_set_cutouts).  cutouts: iterable of (transform, shape, action, space), at most GSR_MAX_CUTOUTS, where transform is a Godot
        Transform3D in matrix form -- a (3, 4) array [basis | origin], or (4, 4) -- that maps the unit cube [-1, 1]^3
        (GSR_CUTOUT_BOX) or the unit sphere (GSR_CUTOUT_ELLIPSOID) onto the volume: in Godot world space for GSR_CUTOUT_FRAME, in the
        asset's own Godot space (the space of set_instances' ranges) for GSR_CUTOUT_SOURCE.  action: GSR_CUTOUT_KEEP or
        GSR_CUTOUT_REMOVE.  A splat is kept or removed whole, by its centre.  An empty list switches cutouts off."""
        items = list(cutouts)
        self._cutouts = [(cutout_to_local(t, self.basis_override), int(shape), int(action), int(space)) for t, shape, action, space in items]
        if self._ctx:
            self._apply_cutouts()

    def _apply_cutouts(self) -> None:
        arr = (_lib.GsrCutout * max(1, len(self._cutouts)))()
        for k, (to_local, shape, action, space) in enumerate(self._cutouts):
            arr[k].to_local[:] = [float(v) for v in to_local.T.reshape(12)]
            arr[k].shape, arr[k].action, arr[k].space = shape, action, space
        _lib.check(_lib.lib().gsr_set_cutouts(self._ctx, arr, len(self._cutouts)), "gsr_set_cutouts")

    def _emit_loaded(self):
        self.is_loaded = True
        for cb in self.loaded_callbacks:
            cb()

    def set_framebuffer_external(self, device_ptr: int) -> None:
        _lib.check(_lib.lib().gsr_set_framebuffer_external(self._ctx, C.c_void_p(device_ptr)), "gsr_set_framebuffer_external")
        self._bind_texture()

    def set_depth_compositing(self, scene_depth_ptr: int | None, depth_out_ptr: int | None) -> None:
        """Composite into the host's 3D scene (include/gsr.h gsr_set_depth_compositing): depth_out_ptr = device float[h*w] that receives
        the splats' linear view depth (None switches the mode off), scene_depth_ptr = optional device float[h*w] linear scene depth
        that hides the splats behind it.  The frame's alpha becomes the coverage."""
        _lib.check(_lib.lib().gsr_set_depth_compositing(self._ctx, C.c_void_p(scene_depth_ptr or None), C.c_void_p(depth_out_ptr or None)),
                   "gsr_set_depth_compositing")

    def set_motion_vectors(self, motion_out_ptr: int | None) -> None:
        """Write the splats' per-pixel screen motion since the previous frame (include/gsr.h gsr_set_motion_vectors): motion_out_ptr =
        device float[h*w*2], (x, y) in pixels per pixel, previous position minus current; None switches it off.  Needs depth
        compositing (set_depth_compositing first)."""
        _lib.check(_lib.lib().gsr_set_motion_vectors(self._ctx, C.c_void_p(motion_out_ptr or None)), "gsr_set_motion_vectors")

    def reset_motion(self) -> None:
        """A camera cut: the next frame reports no motion (include/gsr.h gsr_reset_motion)."""
        _lib.check(_lib.lib().gsr_reset_motion(self._ctx), "gsr_reset_motion")

    def set_splat_ids(self, ids_out_ptr: int | None) -> None:
        """Write, per pixel, the splat and the instance that dominate the blend (include/gsr.h gsr_set_splat_ids): ids_out_ptr = device
        uint32[h*w*2], (drawn id v, instance k) per pixel, GSR_NO_ID where no splat covers it; None switches it off.  Needs depth
        compositing (set_depth_compositing first).  splat_sources maps the array to source splat indices."""
        _lib.check(_lib.lib().gsr_set_splat_ids(self._ctx, C.c_void_p(ids_out_ptr or None)), "gsr_set_splat_ids")

    def set_splat_contribution(self, accum_ptr: int | None) -> None:
        """Accumulate every splat's blend weight over the frames rendered from now on (include/gsr.h gsr_set_splat_contribution):
        accum_ptr = a zeroed device array of max_splats 32-byte gsr_splat_contribution records (e.g. a torch uint8 tensor of
        32 * max_splats bytes), one per source slot; None switches it off.  Needs depth compositing (set_depth_compositing first), and
        neither motion vectors nor splat IDs.  read_splat_contribution decodes a downloaded copy; the GSR_PROP_CONTRIBUTION ..
        properties select and histogram by it."""
        _lib.check(_lib.lib().gsr_set_splat_contribution(self._ctx, C.c_void_p(accum_ptr or None), self._max_splats if accum_ptr else 0),
                   "gsr_set_splat_contribution")

    def reset_splat_contribution(self) -> None:
        """Zero the contribution buffer and the frame counter, ordered between the frames enqueued before and after the call."""
        _lib.check(_lib.lib().gsr_reset_splat_contribution(self._ctx), "gsr_reset_splat_contribution")

    def splat_contribution_frames(self) -> int:
        """The frames accumulated since the last set or reset; a frame that overflowed the duplicate capacity is not (synchronises)."""
        n = C.c_uint32(0)
        _lib.check(_lib.lib().gsr_splat_contribution_frames(self._ctx, C.byref(n)), "gsr_splat_contribution_frames")
        return int(n.value)

    def splat_sources(self, ids: np.ndarray) -> np.ndarray:
        """The source splat index of every pixel of an (h, w, 2) array read back from set_splat_ids' plane, under the current instance
        layout (set_instances): GSR_NO_ID where the pixel has no splat.  Valid for frames rendered with that layout."""
        return splat_sources(ids, self._instance_ranges)

    def set_instances(self, instances) -> None:
        """Draw placed, moving and repeated ranges of the splat buffer in one sorted frame (include/gsr.h gsr_set_instances).
        instances: iterable of (first, count, transform), where transform is a Godot Transform3D in matrix form -- a (3, 4) array
        [basis | origin] whose basis columns are the x, y, z axes (a (4, 4) matrix is accepted too) -- mapping the range's splats,
        placed as the whole cloud is placed today, to their Godot world position.  An empty list switches instancing off.
        Calling it every frame with the same (first, count) sequence only moves the instances (no host synchronisation)."""
        items = list(instances)
        arr = (_lib.GsrInstance * max(1, len(items)))()
        for k, (first, count, transform) in enumerate(items):
            arr[k].first, arr[k].count = int(first), int(count)
            arr[k].to_frame[:] = [float(v) for v in godot_to_frame(transform, self.basis_override).T.reshape(12)]
        _lib.check(_lib.lib().gsr_set_instances(self._ctx, arr, len(items)), "gsr_set_instances")
        self._instance_ranges = [(int(first), int(count)) for first, count, _ in items] if items else None

    def set_instance_appearance(self, appearance) -> None:
        """Show, hide, fade, tint and shorten the instances of set_instances, per frame and without a host synchronisation (include/gsr.h
        gsr_set_instance_appearance).  appearance: one (tint, opacity, draw_count) per instance -- tint an (r, g, b) factor on the
        splat colour, opacity a factor in [0, 1] on the stored splat opacity (0 hides the instance), draw_count the number of
        leading splats of the range to draw (None: all of them) -- or None for the default everywhere.  Like the instances it
        survives a texture_size change; set_instances with a new (first, count) sequence resets it."""
        if appearance is None:
            _lib.check(_lib.lib().gsr_set_instance_appearance(self._ctx, None, 0), "gsr_set_instance_appearance")
            return
        arr = pack_instance_appearance(appearance)
        _lib.check(_lib.lib().gsr_set_instance_appearance(self._ctx, arr, len(arr)), "gsr_set_instance_appearance")

    # ---- splat selection (include/gsr.h "Splat selection"): per-splat selected / hidden masks set on the GPU ----
    def select_polygon(self, xy, op: int = _lib.GSR_SELECT_SET, instance: int = -1) -> None:
        """Select the splats whose centres the current camera (update_camera_matrices) projects inside a screen lasso or rectangle: xy =
        (n, 2) pixel positions (column, row) at the current texture size, 3 <= n <= GSR_MAX_SELECT_VERTICES.  instance = -1 tests every
        splat, k only instance k's range at its current transform.  op: GSR_SELECT_SET / _ADD / _SUBTRACT / _TOGGLE."""
        if self.camera_push_constants is None:
            self.update_camera_matrices()
        v = np.ascontiguousarray(xy, dtype=np.float32).reshape(-1, 2)
        fp = C.POINTER(C.c_float)
        _lib.check(_lib.lib().gsr_select_polygon(self._ctx, self.camera_push_constants.ctypes.data_as(fp), float(self.model_scale[0]),
                                                 int(instance), v.ctypes.data_as(fp), v.shape[0], int(op)), "gsr_select_polygon")

    def select_volume(self, transform, shape: int, space: int = _lib.GSR_CUTOUT_FRAME, op: int = _lib.GSR_SELECT_SET,
                      instance: int = -1) -> None:
        """Select the splats whose centres lie in a box or ellipsoid given like set_cutouts' volumes (a Godot Transform3D of the unit
        shape, in world space for GSR_CUTOUT_FRAME, in the asset's space for GSR_CUTOUT_SOURCE)."""
        vol = _lib.GsrCutout()
        vol.to_local[:] = [float(x) for x in cutout_to_local(transform, self.basis_override).T.reshape(12)]
        vol.shape, vol.action, vol.space = int(shape), _lib.GSR_CUTOUT_KEEP, int(space)
        _lib.check(_lib.lib().gsr_select_volume(self._ctx, C.byref(vol), float(self.model_scale[0]), int(instance), int(op)),
                   "gsr_select_volume")

    def select_ids(self, ids_ptr: int, rect=None, op: int = _lib.GSR_SELECT_SET) -> None:
        """"Select what you see": the splats of every pixel of rect = (x0, y0, x1, y1) (None: the whole frame) of a device ID plane
        written by set_splat_ids."""
        w, h = self._texture_size
        x0, y0, x1, y1 = (0, 0, w, h) if rect is None else (int(r) for r in rect)
        _lib.check(_lib.lib().gsr_select_ids(self._ctx, C.c_void_p(ids_ptr), x0, y0, x1, y1, int(op)), "gsr_select_ids")

    def select_all(self, op: int = _lib.GSR_SELECT_SET) -> None:
        """SET: select every splat; SUBTRACT: select none; TOGGLE: invert the selection."""
        _lib.check(_lib.lib().gsr_select_all(self._ctx, int(op)), "gsr_select_all")

    def hide_selection(self) -> None:
        _lib.check(_lib.lib().gsr_hide_selection(self._ctx), "gsr_hide_selection")

    def unhide_all(self) -> None:
        _lib.check(_lib.lib().gsr_unhide_all(self._ctx), "gsr_unhide_all")

    def clear_splat_masks(self) -> None:
        """No splat selected or hidden, and the masks out of use: frames take their usual kernels again."""
        _lib.check(_lib.lib().gsr_clear_splat_masks(self._ctx), "gsr_clear_splat_masks")

    def set_selection_style(self, rgb, strength: float) -> None:
        """Highlight of selected splats: colour * (1 - strength) + rgb * strength (strength 0: no highlight)."""
        c = (C.c_float * 3)(*[float(x) for x in rgb])
        _lib.check(_lib.lib().gsr_set_selection_style(self._ctx, c, float(strength)), "gsr_set_selection_style")

    def splat_masks(self) -> tuple[np.ndarray, np.ndarray]:
        """(hidden, selected): numpy bool arrays over the source splats (synchronises).  The kept cloud is table[~hidden]."""
        n = self._max_splats
        words = (n + 31) // 32
        hid, sel = np.zeros(words, dtype=np.uint32), np.zeros(words, dtype=np.uint32)
        u32p = C.POINTER(C.c_uint32)
        _lib.check(_lib.lib().gsr_get_splat_masks(self._ctx, hid.ctypes.data_as(u32p), sel.ctypes.data_as(u32p), words), "gsr_get_splat_masks")
        return unpack_mask(hid, n), unpack_mask(sel, n)

    def set_splat_masks(self, hidden, selected) -> None:
        """Restore masks read with splat_masks (undo): bool arrays over the source splats, never both True for one splat."""
        n = self._max_splats
        hid, sel = pack_mask(hidden, n), pack_mask(selected, n)
        u32p = C.POINTER(C.c_uint32)
        _lib.check(_lib.lib().gsr_set_splat_masks(self._ctx, hid.ctypes.data_as(u32p), sel.ctypes.data_as(u32p), hid.size), "gsr_set_splat_masks")

    def selection_counts(self) -> tuple[int, int]:
        """(selected, hidden) splat counts (synchronises)."""
        s, h = C.c_uint64(0), C.c_uint64(0)
        _lib.check(_lib.lib().gsr_splat_mask_counts(self._ctx, C.byref(s), C.byref(h)), "gsr_splat_mask_counts")
        return int(s.value), int(h.value)

    # ---- splat property selection (include/gsr.h "Splat property selection") ----
    def select_where(self, filters, op: int = _lib.GSR_SELECT_SET, instance: int = -1) -> None:
        """Select the splats of the cloud (instance = -1) or of instance k's range, within [0, num_splats), that pass ALL filters:
        each a splat_filter() or a (property, lo, hi[, rgb]) tuple, passing iff lo <= value <= hi (a NaN value never passes), 1 to
        GSR_MAX_SPLAT_FILTERS of them.  Properties (GSR_PROP_*) come from the stored words: opacity, size (the sum of the squared
        scales), volume (their product), isotropy (1 for a sphere, towards 0 for needles and discs) and the squared distance of the DC
        colour from rgb.  A vacant slot is never selected.  op: GSR_SELECT_SET / _ADD / _SUBTRACT / _TOGGLE; hidden splats stay
        unselected."""
        fs = [f if isinstance(f, _lib.GsrSplatFilter) else splat_filter(*f) for f in filters]
        arr = (_lib.GsrSplatFilter * max(1, len(fs)))(*fs)
        _lib.check(_lib.lib().gsr_select_where(self._ctx, arr, len(fs), int(instance), int(op)), "gsr_select_where")

    def select_neighborhood(self, mode: int, radius: float, count: int = 1, op: int = _lib.GSR_SELECT_SET, instance: int = -1) -> dict:
        """Select splats by their neighbourhood (include/gsr.h "Splat neighbourhood selection"): participants are the splats of the cloud
        (instance = -1) or of instance k's range that are not hidden and have a finite position; two are neighbours within `radius`
        (source units).  mode: GSR_NEIGHBOR_SPARSE (fewer than `count` neighbours), _GROW (selected or next to a selected splat),
        _CONNECTED (the clusters holding a selected splat), _SMALL_CLUSTERS (clusters of fewer than `count` splats); op as every
        select_*.  Returns the stats: participants, inside, candidates, clusters, largest_cluster.  Synchronises at most twice."""
        q = _lib.GsrNeighborhood(int(mode), float(radius), int(count), int(instance))
        st = _lib.GsrNeighborhoodStats()
        _lib.check(_lib.lib().gsr_select_neighborhood(self._ctx, C.byref(q), int(op), C.byref(st)), "gsr_select_neighborhood")
        return {k: int(getattr(st, k)) for k, _ in _lib.GsrNeighborhoodStats._fields_}

    def splat_histogram(self, property: int, edges, scope: int = _lib.GSR_HISTOGRAM_KEPT, instance: int = -1, rgb=None):
        """Histogram of a property (GSR_PROP_*; rgb for GSR_PROP_COLOR_DISTANCE) over the splats that are not hidden
        (GSR_HISTOGRAM_KEPT) or that are selected (GSR_HISTOGRAM_SELECTED), of the cloud or of instance k's range.  edges: bins + 1
        finite, strictly increasing values.  Returns (counts, below, above, nan, (min, max)): counts[i] of edges[i] <= v < edges[i + 1]
        (the last bin also takes v == edges[-1]), the counts below edges[0], above edges[-1] and of NaN values, and the least and
        greatest non-NaN value ((inf, -inf) when there is none).  Synchronises once."""
        e = np.ascontiguousarray(edges, dtype=np.float32).reshape(-1)
        bins = max(e.size - 1, 0)
        counts = np.zeros(bins + 3, dtype=np.uint64)
        mm = np.zeros(2, dtype=np.float32)
        f = splat_filter(property, rgb=rgb)
        fp = C.POINTER(C.c_float)
        _lib.check(_lib.lib().gsr_splat_histogram(self._ctx, C.byref(f), int(instance), int(scope), e.ctypes.data_as(fp), bins,
                                                  counts.ctypes.data_as(C.POINTER(C.c_uint64)), mm.ctypes.data_as(fp)),
                   "gsr_splat_histogram")
        return counts[:bins], int(counts[bins]), int(counts[bins + 1]), int(counts[bins + 2]), (float(mm[0]), float(mm[1]))

    # ---- splat transform edits (include/gsr.h "Splat transform edits") ----
    def transform_selection(self, transform, space: int = _lib.GSR_CUTOUT_FRAME, instance: int = -1, snapshot_ptr: int | None = None) -> None:
        """Move, rotate, scale or mirror the selected splats in the store.  transform: a frame-space (3, 4) [B | u] (godot_to_frame
        converts a Godot Transform3D).  GSR_CUTOUT_SOURCE applies it to the stored positions as given; GSR_CUTOUT_FRAME applies it in
        frame space as instance `instance` draws the splats (-1: no instance), with the current model_scale.  snapshot_ptr: a device
        snapshot from copy_splat_store to read instead of the store (a drag re-applies its growing transform to the mouse-down state)."""
        T = np.asarray(transform, dtype=np.float64)
        if T.shape == (4, 4):
            T = T[:3]
        assert T.shape == (3, 4), T.shape
        if int(space) == _lib.GSR_CUTOUT_SOURCE:
            m = T.astype(np.float32)
        else:
            A, tk = np.eye(3), np.zeros(3)
            if instance >= 0:
                x = self.debug_copy(_lib.GSR_BUF_INSTANCES, 24 * len(self._instance_ranges), np.float32)
                k = x[24 * instance:24 * instance + 12].astype(np.float64).reshape(4, 3).T
                A, tk = k[:, :3], k[:, 3]
            m = compose_frame_edit(T, A, tk, float(self.model_scale[0]))
        ts = np.ascontiguousarray(m.T.reshape(12), dtype=np.float32)
        _lib.check(_lib.lib().gsr_transform_selection(self._ctx, ts.ctypes.data_as(C.POINTER(C.c_float)),
                                                      None if snapshot_ptr is None else C.c_void_p(snapshot_ptr)), "gsr_transform_selection")

    def recolor_selection(self, edit: _lib.GsrColorEdit, snapshot_ptr: int | None = None) -> None:
        """Recolour, fade or flatten the selected splats in the store (include/gsr.h "Splat colour edits"); color_edit() builds `edit`.
        snapshot_ptr: a device snapshot from copy_splat_store to read instead of the store (a slider drag re-applies its growing edit
        to the mouse-down state)."""
        _lib.check(_lib.lib().gsr_recolor_selection(self._ctx, C.byref(edit), None if snapshot_ptr is None else C.c_void_p(snapshot_ptr)),
                   "gsr_recolor_selection")

    # ---- splat delete and duplicate (include/gsr.h "Splat delete and duplicate"); each synchronises once ----
    def delete_hidden(self) -> int:
        """Compact the hidden splats out of [0, num_splats): the kept splats move down in order and the count k of them becomes
        num_splats.  Returns k.  The splat at s moves to delete_remap(hidden)[s] (hidden as splat_masks() read it before the call)."""
        k = C.c_uint64(0)
        _lib.check(_lib.lib().gsr_delete_hidden(self._ctx, C.byref(k)), "gsr_delete_hidden")
        return int(k.value)

    def duplicate_selection(self) -> int:
        """Append copies of the selected splats of [0, num_splats) behind it and select exactly the copies.  Returns their count."""
        s = C.c_uint64(0)
        _lib.check(_lib.lib().gsr_duplicate_selection(self._ctx, C.byref(s)), "gsr_duplicate_selection")
        return int(s.value)

    def set_splat_count(self, n: int) -> None:
        """Set num_splats (undo of delete_hidden / duplicate_selection, after restore_splat_store and set_splat_masks)."""
        _lib.check(_lib.lib().gsr_set_splat_count(self._ctx, int(n)), "gsr_set_splat_count")

    def splat_store_bytes(self) -> int:
        return int(_lib.lib().gsr_splat_store_bytes(self._ctx))

    def copy_splat_store(self, ptr: int) -> None:
        """Snapshot the whole store into device or page-locked host memory of splat_store_bytes() bytes (enqueued; no host sync)."""
        _lib.check(_lib.lib().gsr_copy_splat_store(self._ctx, C.c_void_p(ptr)), "gsr_copy_splat_store")

    def restore_splat_store(self, ptr: int) -> None:
        """Write a snapshot of copy_splat_store back (undo of an edit, together with set_splat_masks)."""
        _lib.check(_lib.lib().gsr_restore_splat_store(self._ctx, C.c_void_p(ptr)), "gsr_restore_splat_store")

    def kept_table(self) -> np.ndarray:
        """The edited cloud as a float32 3DGS vertex table (degree_properties of the store's degree, normals 0): the splats of
        [0, num_splats) whose hidden bit is 0, read from the device store (synchronises).  PlyFile.from_array(table).save(path) writes
        it."""
        stride = self._plane_stride()
        store = np.empty((self.splat_store_bytes() // (16 * stride), stride, 4), dtype=np.float32)
        self.copy_splat_store(store.ctypes.data)   # pageable memory: the copy has landed when the call returns
        n = int(self.stats().num_splats)
        hidden, _ = self.splat_masks()
        bands = self._sh_bands if self._sh_bands else 4
        return store_to_table(store, n, bands, bool(self._flags & _lib.GSR_FLAG_SH_HALF), hidden[:n])

    def export_ply(self, scope: int = _lib.GSR_EXPORT_KEPT, sh_degree: int = -1) -> PlyFile:
        """The edited cloud exported on the GPU (include/gsr.h "Splat export"): the splats of [0, num_splats) that are not hidden
        (GSR_EXPORT_KEPT) or that are selected (GSR_EXPORT_SELECTED), vacant slots skipped, as the float32 rows of a 3DGS PLY of SH
        degree sh_degree (-1: the stored degree), in store order, with their degree_properties names.  r.export_ply().save(path)
        writes the file.  Synchronises twice (the count, then the rows)."""
        from .ply_file import degree_properties
        L, rows = _lib.lib(), C.c_uint64(0)
        _lib.check(L.gsr_export_ply(self._ctx, int(scope), int(sh_degree), None, 0, C.byref(rows)), "gsr_export_ply")
        degree = (self._sh_bands if self._sh_bands else 4) - 1 if int(sh_degree) < 0 else int(sh_degree)
        names = degree_properties(degree)
        table = np.empty((rows.value, len(names)), dtype=np.float32)
        if rows.value:
            _lib.check(L.gsr_export_ply(self._ctx, int(scope), int(sh_degree), C.c_void_p(table.ctypes.data), table.shape[0], C.byref(rows)),
                       "gsr_export_ply")
        return PlyFile.from_array(table, names)

    def export_compressed_ply(self, scope: int = _lib.GSR_EXPORT_KEPT, sh_degree: int = -1,
                              order: int = _lib.GSR_COMPRESS_MORTON) -> CompressedPlyFile:
        """The edited cloud exported on the GPU as a SuperSplat compressed PLY (include/gsr.h "Compressed PLY"): the splats of export_ply's
        scope with a finite position, in Morton order (GSR_COMPRESS_MORTON, the smaller chunk ranges) or store order
        (GSR_COMPRESS_STORE_ORDER, the rows of export_ply), SH degree sh_degree (-1: the stored degree).  r.export_compressed_ply().save(path)
        writes the file.  Synchronises twice (the count, then the file)."""
        L, rows = _lib.lib(), C.c_uint64(0)
        _lib.check(L.gsr_export_compressed_ply(self._ctx, int(scope), int(sh_degree), int(order), None, C.byref(rows)), "gsr_export_compressed_ply")
        degree = (self._sh_bands if self._sh_bands else 4) - 1 if int(sh_degree) < 0 else int(sh_degree)
        n = rows.value
        chunks = np.empty(((n + _lib.GSR_COMPRESSED_CHUNK - 1) // _lib.GSR_COMPRESSED_CHUNK, 18), dtype=np.float32)
        packed = np.empty((n, 4), dtype=np.uint32)
        sh = np.empty((n, 3 * ((degree + 1) ** 2 - 1)), dtype=np.uint8) if degree > 0 else None
        if n:
            dst = _lib.GsrCompressedPly(chunks.ctypes.data, packed.ctypes.data, sh.ctypes.data if sh is not None else None, n, chunks.shape[0],
                                        degree, 18)
            _lib.check(L.gsr_export_compressed_ply(self._ctx, int(scope), int(sh_degree), int(order), C.byref(dst), C.byref(rows)),
                       "gsr_export_compressed_ply")
        return CompressedPlyFile.from_arrays(chunks, packed, sh, degree)

    def upload_compressed_ply(self, cply: CompressedPlyFile, first: int = 0, creation_time: float = 0.0) -> None:
        """Device decode of a compressed PLY into splats [first, first + cply.size) (include/gsr.h gsr_upload_compressed_ply)."""
        if not self._ctx:
            raise RuntimeError("init_gpu() first")
        chunks = np.ascontiguousarray(cply.chunks, dtype=np.float32)
        packed = np.ascontiguousarray(cply.packed, dtype=np.uint32)
        sh = np.ascontiguousarray(cply.sh, dtype=np.uint8) if cply.sh_degree > 0 else None
        src = _lib.GsrCompressedPly(chunks.ctypes.data, packed.ctypes.data, sh.ctypes.data if sh is not None else None, cply.size,
                                    chunks.shape[0], cply.sh_degree, chunks.shape[1])
        _lib.check(_lib.lib().gsr_upload_compressed_ply(self._ctx, C.byref(src), int(first), float(creation_time)), "gsr_upload_compressed_ply")
        self.num_splats_loaded[0] = max(self.num_splats_loaded[0], int(first) + cply.size)

    def _plane_stride(self) -> int:
        return (self._max_splats + 255) // 256 * 256

    def render_raw(self, vp32: np.ndarray, uniforms32: bytes, heatmap: float = 0.0, host_ptr: int | None = None,
                   asynchronous: bool = True, rgb_only: bool = False, out_format: int | None = None) -> None:
        """rasterize() with pre-packed push constants / uniform block (bench hot loop).  out_format: GSR_OUT_* of the host frame
        (| GSR_OUT_SRGB_TO_LINEAR); rgb_only is shorthand for GSR_OUT_RGB32F (alpha is constant 1.0 and stays on the device)."""
        L = _lib.lib()
        fmt = _lib.GSR_OUT_RGB32F if (rgb_only and out_format is None) else (out_format or _lib.GSR_OUT_RGBA32F)
        vpp = vp32.ctypes.data_as(C.POINTER(C.c_float))
        hp = None if host_ptr is None else C.c_void_p(host_ptr)
        if not asynchronous:
            assert fmt == _lib.GSR_OUT_RGBA32F, "gsr_render returns the RGBA32F frame"
            _lib.check(L.gsr_render(self._ctx, vpp, uniforms32, float(heatmap), hp), "gsr_render")
        else:
            _lib.check(L.gsr_render_async_fmt(self._ctx, vpp, uniforms32, float(heatmap), hp, int(fmt)), "gsr_render_async_fmt")

    def debug_pipeline(self, overlap: int) -> None:
        """gsr_debug_pipeline: 1 / 0 = front/back overlap of consecutive frames on / off, -1 = automatic (include/gsr.h)."""
        _lib.check(_lib.lib().gsr_debug_pipeline(self._ctx, int(overlap)), "gsr_debug_pipeline")

    def set_stream(self, cuda_stream: int) -> None:
        _lib.check(_lib.lib().gsr_set_stream(self._ctx, C.c_void_p(cuda_stream)), "gsr_set_stream")

    def set_band(self, row_begin: int, row_end: int) -> None:
        _lib.check(_lib.lib().gsr_set_band(self._ctx, row_begin, row_end), "gsr_set_band")

    def set_row_interleave(self, rem: int, mod: int) -> None:
        """Own the tile rows with row % mod == rem (balanced multi-GPU sharding, fast mode; see include/gsr.h)."""
        _lib.check(_lib.lib().gsr_set_row_interleave(self._ctx, rem, mod), "gsr_set_row_interleave")

    def band_sync_word_ptr(self) -> int:
        return int(_lib.lib().gsr_band_sync_word(self._ctx) or 0)

    def band_fixup(self) -> None:
        _lib.check(_lib.lib().gsr_band_fixup(self._ctx), "gsr_band_fixup")

    def cleanup_gpu(self) -> None:  # rasterizer.gd:116-120
        self.should_terminate_thread[0] = True
        if self._ctx:
            _lib.lib().gsr_destroy(self._ctx)
            self._ctx = C.c_void_p(None)
            self._instance_ranges = None
        if self.render_texture:
            self.render_texture.device_ptr = 0

    # ---- rasterize (rasterizer.gd:122-160) ----
    def uniforms_bytes(self, time: float | None = None) -> bytes:
        cam_pos = self.basis_override.T @ np.asarray(self.camera.global_position, dtype=np.float32)
        w, h = self._texture_size
        t = self.ticks() if time is None else time
        buf = np.zeros(8, dtype=np.float32)
        buf[0], buf[1], buf[2], buf[3] = -cam_pos[0], -cam_pos[1], cam_pos[2], self.model_scale[0]
        buf[6] = t
        raw = bytearray(buf.tobytes())
        raw[16:24] = np.array([w, h], dtype=np.int32).tobytes()
        return bytes(raw)

    def rasterize(self, time: float | None = None, out_host: np.ndarray | None = None, asynchronous: bool = False) -> None:
        if not self._ctx:
            self.init_gpu()
        if self.camera_push_constants is None:
            self.update_camera_matrices()
        u = self.uniforms_bytes(time)
        vp = self.camera_push_constants
        fn = _lib.lib().gsr_render_async if asynchronous else _lib.lib().gsr_render
        outp = None if out_host is None else C.c_void_p(out_host.ctypes.data)
        _lib.check(fn(self._ctx, vp.ctypes.data_as(C.POINTER(C.c_float)), u, float(self.should_enable_heatmap[0]), outp),
                   "gsr_render")

    def sync(self) -> None:
        _lib.check(_lib.lib().gsr_sync(self._ctx), "gsr_sync")

    def readback_async(self, host_ptr: int, rgb_only: bool = False, out_format: int | None = None) -> None:
        fmt = _lib.GSR_OUT_RGB32F if (rgb_only and out_format is None) else (out_format or _lib.GSR_OUT_RGBA32F)
        _lib.check(_lib.lib().gsr_readback_async(self._ctx, C.c_void_p(host_ptr), int(fmt)), "gsr_readback_async")

    def present_device(self, device_ptr: int, out_format: int = 0) -> None:
        """Converted copy of the last frame into caller-owned device memory (imported external image / torch tensor)."""
        _lib.check(_lib.lib().gsr_present_device(self._ctx, C.c_void_p(device_ptr), int(out_format)), "gsr_present_device")

    def peer_export(self) -> bytes:
        """Presenting rank: CUDA-IPC handles (128 bytes) of its two frames."""
        buf = (C.c_ubyte * 128)()
        _lib.check(_lib.lib().gsr_peer_export_framebuffers(self._ctx, buf), "gsr_peer_export_framebuffers")
        return bytes(buf)

    def peer_import(self, handles: bytes) -> None:
        buf = (C.c_ubyte * 128).from_buffer_copy(handles)
        _lib.check(_lib.lib().gsr_peer_import_framebuffers(self._ctx, buf), "gsr_peer_import_framebuffers")

    # ---- multi-GPU shard group (include/gsr.h gsr_group_*): NCCL-free frame path over NVLink peer memory ----
    def group_export(self) -> bytes:
        buf = (C.c_ubyte * _lib.GSR_GROUP_BLOB_BYTES)()
        _lib.check(_lib.lib().gsr_group_export(self._ctx, buf), "gsr_group_export")
        return bytes(buf)

    def group_attach(self, rank: int, world: int, blobs: bytes) -> None:
        assert len(blobs) == world * _lib.GSR_GROUP_BLOB_BYTES
        buf = (C.c_ubyte * len(blobs)).from_buffer_copy(blobs)
        _lib.check(_lib.lib().gsr_group_attach(self._ctx, int(rank), int(world), buf), "gsr_group_attach")

    def group_set_present(self, rows_local: bool) -> None:
        _lib.check(_lib.lib().gsr_group_set_present(self._ctx, int(bool(rows_local))), "gsr_group_set_present")

    def readback_rows_async(self, host_frame_ptr: int) -> None:
        _lib.check(_lib.lib().gsr_readback_rows_async(self._ctx, C.c_void_p(host_frame_ptr)), "gsr_readback_rows_async")

    def group_detach(self) -> None:
        _lib.check(_lib.lib().gsr_group_detach(self._ctx), "gsr_group_detach")

    def stream_join(self) -> None:
        """Make the render stream wait for the pipelined read-back copies enqueued so far."""
        _lib.check(_lib.lib().gsr_stream_join(self._ctx), "gsr_stream_join")

    # ---- get_splat_position (rasterizer.gd:162-171) ----
    def get_splat_position(self, screen_position) -> np.ndarray:
        s = self.render_scale[0]
        tile = (int(screen_position[0] * s) // TILE_SIZE, int(screen_position[1] * s) // TILE_SIZE)
        tile_id = tile[1] * self.tile_dims[0] + tile[0]
        out = (C.c_float * 4)()
        rc = _lib.lib().gsr_pick(self._ctx, tile_id & 0xFFFFFFFF, float(self.should_enable_heatmap[0]), out)
        if rc == _lib.GSR_ERR_STATE:   # no frame rasterized yet: the reference reads its zero-initialised buffer -> Vector3.INF
            return VECTOR3_INF.copy()
        _lib.check(rc, "gsr_pick")
        if out[3] == 0:
            return VECTOR3_INF.copy()
        v = np.array([-out[0], -out[1], out[2]], dtype=np.float32)
        return np.linalg.inv(self.basis_override.T.astype(np.float64)).astype(np.float32) @ v

    # ---- update_camera_matrices (rasterizer.gd:175-195) ----
    def update_camera_matrices(self) -> bool:
        cam = np.asarray(self.camera.get_camera_transform(), dtype=np.float32).reshape(4, 4)
        bo = self.basis_override  # rows are columns x,y,z
        if np.array_equal(bo, np.eye(3, dtype=np.float32)):
            view = cam.reshape(16)
        else:
            B = bo.T.astype(np.float32)  # matrix form
            basis = (B @ cam[:3, :3].T).T.astype(np.float32)
            origin = (B @ cam[3, :3]).astype(np.float32)
            view = transform_to_projection(basis, origin)
        proj = np.asarray(self.camera.get_camera_projection(), dtype=np.float32)
        if (self.camera_transform is None or not np.array_equal(view, self.camera_transform)
                or not np.array_equal(proj, self.camera_projection)):
            self.camera_transform, self.camera_projection = view, proj
            # a GSR_FLAG_ORTHOGRAPHIC context sees the projection's own w row (the reference packing forces the perspective one);
            # for perspective and frustum matrices both give the same bytes
            self.camera_push_constants = pack_camera_push_constants(view, proj, keep_w_row=bool(self._flags & _lib.GSR_FLAG_ORTHOGRAPHIC))
            return True
        return False

    # ---- debug / stats (main.gd:93-119) ----
    def stats(self) -> _lib.GsrStats:
        st = _lib.GsrStats()
        _lib.check(_lib.lib().gsr_get_stats(self._ctx, C.byref(st)), "gsr_get_stats")
        return st

    def frame_history(self, max_frames: int = _lib.GSR_HISTORY_FRAMES) -> list:
        """Per-frame GPU timestamps + counters of the most recent frames (main.gd:106-119)."""
        n = min(max_frames, _lib.GSR_HISTORY_FRAMES)
        buf = (_lib.GsrFrameRecord * n)()
        got = C.c_uint32(0)
        _lib.check(_lib.lib().gsr_get_frame_history(self._ctx, n, buf, C.byref(got)), "gsr_get_frame_history")
        return [buf[i] for i in range(got.value)]

    def read_framebuffer(self) -> np.ndarray:
        w, h = self._texture_size
        out = np.empty((h, w, 4), dtype=np.float32)
        _lib.check(_lib.lib().gsr_debug_copy(self._ctx, _lib.GSR_BUF_FRAMEBUFFER, C.c_void_p(out.ctypes.data), out.nbytes),
                   "gsr_debug_copy")
        return out

    def debug_copy(self, which: int, count: int, dtype) -> np.ndarray:
        out = np.empty(count, dtype=dtype)
        _lib.check(_lib.lib().gsr_debug_copy(self._ctx, which, C.c_void_p(out.ctypes.data), out.nbytes), "gsr_debug_copy")
        return out

    def keep_unsorted(self, enable: bool = True) -> None:
        _lib.check(_lib.lib().gsr_debug_keep_unsorted(self._ctx, int(enable)), "gsr_debug_keep_unsorted")


def pack_instance_appearance(appearance):
    """[(tint, opacity, draw_count | None), ...] -> a ctypes array of gsr_instance_appearance (None: GSR_DRAW_ALL, every splat)."""
    items = list(appearance)
    arr = (_lib.GsrInstanceAppearance * len(items))()
    for k, (tint, opacity, draw_count) in enumerate(items):
        arr[k].tint[:] = [float(v) for v in tint]
        arr[k].opacity = float(opacity)
        arr[k].draw_count = _lib.GSR_DRAW_ALL if draw_count is None else int(draw_count)
    return arr


def splat_sources(ids: np.ndarray, ranges=None) -> np.ndarray:
    """(h, w, 2) uint32 (v, k) of gsr_set_splat_ids -> (h, w) uint32 source splat indices.  ranges: the (first, count) per instance of
    the frame's gsr_set_instances layout, or None without instances (the source is v).  Instance k's drawn ids start at warp
    w_k = sum of ceil(count_j / 32) over j < k, so v maps to first_k + (v - 32 w_k).  GSR_NO_ID stays GSR_NO_ID."""
    ids = np.asarray(ids, dtype=np.uint32)
    assert ids.shape[-1] == 2, ids.shape
    v, k = ids[..., 0], ids[..., 1]
    out = np.full(v.shape, _lib.GSR_NO_ID, dtype=np.uint32)
    hit = v != _lib.GSR_NO_ID
    if not ranges:
        out[hit] = v[hit]
        return out
    counts = np.array([int(c) for _, c in ranges], dtype=np.int64)
    w0 = np.concatenate([[0], np.cumsum((counts + 31) // 32)[:-1]])
    first = np.array([int(f) for f, _ in ranges], dtype=np.int64)
    kk = k[hit].astype(np.int64)
    out[hit] = (first[kk] + (v[hit].astype(np.int64) - 32 * w0[kk])).astype(np.uint32)
    return out


def pack_mask(mask, n: int) -> np.ndarray:
    """A bool array over n splats -> the ceil(n / 32) uint32 words of include/gsr.h (splat s = bit s & 31 of word s >> 5)."""
    m = np.asarray(mask, dtype=bool).reshape(-1)
    assert m.size == n, (m.size, n)
    words = (n + 31) // 32
    bits = np.zeros(words * 32, dtype=bool)
    bits[:n] = m
    return np.packbits(bits, bitorder="little").view("<u4").astype(np.uint32)


def unpack_mask(words: np.ndarray, n: int) -> np.ndarray:
    """The inverse of pack_mask: uint32 words -> a bool array over n splats."""
    return np.unpackbits(np.ascontiguousarray(words, dtype="<u4").view(np.uint8), bitorder="little")[:n].astype(bool)


CONTRIBUTION_DTYPE = np.dtype([("weight", "<u8"), ("pixels", "<u8"), ("peak", "<f4"), ("views", "<u4"), ("last_frame", "<u4"),
                               ("pad", "<u4")])   # gsr_splat_contribution


def read_splat_contribution(buf) -> dict:
    """Decode a contribution buffer (gsr_set_splat_contribution) downloaded to the host -- bytes, a uint8 array or a torch tensor on any
    device -- into numpy arrays over the slots: weight (float64, the sum of q(w) / 2^24), pixels, peak and views."""
    if hasattr(buf, "detach"):   # a torch tensor
        buf = buf.detach().cpu().contiguous().view(-1).numpy()
    raw = np.frombuffer(buf, dtype=np.uint8) if isinstance(buf, (bytes, bytearray, memoryview)) else np.ascontiguousarray(buf).view(np.uint8)
    rec = raw.view(CONTRIBUTION_DTYPE)
    return {"weight": rec["weight"].astype(np.float64) * 2.0 ** -24, "pixels": rec["pixels"].copy(), "peak": rec["peak"].copy(),
            "views": rec["views"].copy()}


def splat_filter(property: int, lo: float = -np.inf, hi: float = np.inf, rgb=None) -> _lib.GsrSplatFilter:
    """One gsr_splat_filter: the property (GSR_PROP_*) passes iff lo <= value <= hi; rgb is the reference colour of
    GSR_PROP_COLOR_DISTANCE (default black; ignored by the other properties).  GSR_PROP_CONTRIBUTION, _PEAK_CONTRIBUTION, _VIEWS
    and _CONTRIBUTING_PIXELS read the contribution buffer of set_splat_contribution."""
    f = _lib.GsrSplatFilter()
    f.property, f.lo, f.hi = int(property), float(lo), float(hi)
    f.rgb[:] = [float(x) for x in (rgb if rgb is not None else (0.0, 0.0, 0.0))]
    return f


def delete_remap(hidden, n: int) -> np.ndarray:
    """The new index of every splat of [0, n) after delete_hidden, from the hidden mask read before it: the number of kept splats
    below it (int64), or -1 for a deleted splat."""
    h = np.asarray(hidden, dtype=bool).reshape(-1)[:n]
    rank = np.cumsum(~h, dtype=np.int64) - 1
    return np.where(h, np.int64(-1), rank)


def godot_to_frame(transform, basis_override) -> np.ndarray:
    """A Godot Transform3D (matrix form, (3, 4) [basis | origin] or (4, 4)) -> the (3, 4) float32 [A | t] of gsr_instance.to_frame.

    Frame space is where the uploaded splats, the view matrix and camera_pos live: a Godot world point p sits at F B p in frame
    space, with F = diag(-1, -1, 1) and B = basis_override in matrix form (the convention of update_camera_matrices, uniforms_bytes
    and get_splat_position).  An object placed by T therefore maps splat coordinates by M = F B T B^-1 F.  It is evaluated as
    I + F B (T - I) B^-1 F in float64, so the identity maps to the identity exactly."""
    T = np.asarray(transform, dtype=np.float64)
    if T.shape == (4, 4):
        T = T[:3]
    assert T.shape == (3, 4), T.shape
    D = np.eye(4)
    D[:3] = T
    D -= np.eye(4)
    Fb = np.eye(4)
    Fb[:3, :3] = np.diag([-1.0, -1.0, 1.0]) @ np.asarray(basis_override, dtype=np.float64).T
    M = np.eye(4) + Fb @ D @ np.linalg.inv(Fb)
    return M[:3].astype(np.float32)


def compose_frame_edit(transform, A, t_k, model_scale: float) -> np.ndarray:
    """The source-space [L | t] (3, 4) float32 of a frame-space edit [B | u] of the splats an instance with to_frame [A | t_k] draws:
    it moves frame position A (x * model_scale) + t_k to B (that) + u, so L = A^-1 B A and t = A^-1 (B t_k + u - t_k) / model_scale.
    Composed in float64 and narrowed once."""
    T = np.asarray(transform, dtype=np.float64)
    B, u = T[:, :3], T[:, 3]
    A, t_k = np.asarray(A, dtype=np.float64), np.asarray(t_k, dtype=np.float64)
    Ai = np.linalg.inv(A)
    out = np.empty((3, 4))
    out[:, :3] = Ai @ B @ A
    out[:, 3] = Ai @ (B @ t_k + u - t_k) / model_scale
    return out.astype(np.float32)


REC709_LUMA = (0.2126, 0.7152, 0.0722)


def color_edit(gain=(1.0, 1.0, 1.0), brightness=0.0, contrast=1.0, saturation=1.0, hue=0.0, view_dependence=1.0, opacity=1.0,
               opacity_offset=0.0) -> _lib.GsrColorEdit:
    """The gsr_color_edit of a colour grade, composed in float64 in this order and narrowed once:
      1. channel gain: colour * gain;
      2. saturation: a lerp from the Rec. 709 luma grey (0.2126, 0.7152, 0.0722) . colour to the colour (0: grey, above 1: more
         saturated);
      3. hue: a rotation by `hue` degrees about the grey axis (1, 1, 1);
      4. contrast about 0.5: (colour - 0.5) * contrast + 0.5;
      5. brightness: + brightness.
    view_dependence scales the view-dependent colour (SH bands 1-3; 0 flattens it); opacity and opacity_offset map the stored opacity
    to clamp(o * opacity + opacity_offset, 0, 1).  The defaults give exactly the identity edit."""
    M, b = np.eye(3), np.zeros(3)

    def then(A, t):
        nonlocal M, b
        M, b = A @ M, A @ b + t

    then(np.diag(np.asarray(gain, dtype=np.float64)), np.zeros(3))
    s = float(saturation)
    then(s * np.eye(3) + (1.0 - s) * np.outer(np.ones(3), REC709_LUMA), np.zeros(3))
    a = np.deg2rad(float(hue))
    k = np.ones(3) / np.sqrt(3.0)
    K = np.array([[0.0, -k[2], k[1]], [k[2], 0.0, -k[0]], [-k[1], k[0], 0.0]])
    then(np.cos(a) * np.eye(3) + np.sin(a) * K + (1.0 - np.cos(a)) * np.outer(k, k), np.zeros(3))
    c = float(contrast)
    then(c * np.eye(3), np.full(3, 0.5 * (1.0 - c)))
    then(np.eye(3), np.full(3, float(brightness)))
    e = _lib.GsrColorEdit()
    e.matrix[:] = [float(np.float32(v)) for v in np.concatenate([M.T.reshape(9), b])]
    e.band_scale[:] = [float(view_dependence)] * 3
    e.opacity_scale, e.opacity_offset = float(opacity), float(opacity_offset)
    return e


# logits beyond +-104 give a stored opacity of exactly 0 or 1 in float32, so the export clamps there (a finite PLY value)
_LOGIT_LIMIT = 104.0


def store_to_table(store, n: int, bands: int, half: bool, hidden=None) -> np.ndarray:
    """A store in the layout of GSR_BUF_SPLATS ((planes, plane_stride, 4) float32) -> the float32 3DGS vertex table of its first n
    splats minus the hidden ones, in degree_properties(bands - 1) order with normals 0: the inverse of the ingest (ply_to_soa), in
    float64.  Covariance: eigh(S) = V diag(l) V^T, a column of V flipped when det V < 0, rot = (w, x, y, z) of the rotation V,
    scale_i = log(max(l_i, tiny)) / 2.  Opacity: the logit, clamped to +-104.  Positions and coefficients as stored (binary16 widened),
    f_rest channel-major.  A Mip-Splatting filter is folded into the stored splat already, so no filter_3D property is written."""
    from .ply_file import degree_properties
    s = np.asarray(store, dtype=np.float32)
    keep = np.ones(n, dtype=bool) if hidden is None else ~np.asarray(hidden, dtype=bool)[:n]
    idx = np.flatnonzero(keep)
    m = idx.size
    p0, p1, p2 = s[0, idx].astype(np.float64), s[1, idx].astype(np.float64), s[2, idx].astype(np.float64)
    K = bands * bands
    P = (3 * K + 7) // 8 if half else (3 * K + 3) // 4
    raw = np.ascontiguousarray(s[3:3 + P, idx].transpose(1, 0, 2)).reshape(m, 4 * P)
    if half:
        w = raw.view(np.uint32)
        c = np.stack([w & 0xFFFF, w >> 16], axis=2).reshape(m, 8 * P).astype(np.uint16).view(np.float16).astype(np.float32)
    else:
        c = raw.copy()
    c = c[:, :3 * K].reshape(m, K, 3)
    S = np.empty((m, 3, 3))
    S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1] = p1[:, 0], p1[:, 1], p1[:, 2], p1[:, 3]
    S[:, 1, 2], S[:, 2, 2] = p2[:, 0], p2[:, 1]
    S[:, 1, 0], S[:, 2, 0], S[:, 2, 1] = S[:, 0, 1], S[:, 0, 2], S[:, 1, 2]
    lam, V = np.linalg.eigh(S)
    V[np.linalg.det(V) < 0, :, 0] *= -1.0
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = 0.5 * np.log(np.maximum(lam, np.finfo(np.float64).tiny))
        o = p2[:, 2]
        logit = np.clip(np.log(o) - np.log1p(-o), -_LOGIT_LIMIT, _LOGIT_LIMIT)
    logit = np.where(np.isnan(logit), 0.0, logit)
    names = degree_properties(bands - 1)
    out = np.zeros((m, len(names)), dtype=np.float32)
    col = {name: i for i, name in enumerate(names)}
    out[:, 0:3] = s[0, idx, 0:3]
    out[:, col["f_dc_0"]:col["f_dc_0"] + 3] = c[:, 0, :]
    if K > 1:
        out[:, col["f_rest_0"]:col["f_rest_0"] + 3 * (K - 1)] = c[:, 1:, :].transpose(0, 2, 1).reshape(m, 3 * (K - 1))
    out[:, col["opacity"]] = logit
    out[:, col["scale_0"]:col["scale_0"] + 3] = scale
    out[:, col["rot_0"]:col["rot_0"] + 4] = rotation_quaternion(V)
    return out


def rotation_quaternion(R) -> np.ndarray:
    """(m, 3, 3) proper rotations -> (m, 4) unit quaternions (w, x, y, z), float64 (Shepperd's method: the largest of w, x, y, z first)."""
    R = np.asarray(R, dtype=np.float64)
    tr = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2]
    cand = np.stack([tr, R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]], axis=1)
    k = np.argmax(cand, axis=1)
    q = np.empty((R.shape[0], 4))
    for i in range(4):
        sel = k == i
        r = R[sel]
        if i == 0:
            w = 0.5 * np.sqrt(1.0 + tr[sel])
            f = 0.25 / w
            q[sel] = np.stack([w, (r[:, 2, 1] - r[:, 1, 2]) * f, (r[:, 0, 2] - r[:, 2, 0]) * f, (r[:, 1, 0] - r[:, 0, 1]) * f], axis=1)
        else:
            a, b, cc = i - 1, i % 3, (i + 1) % 3
            v = 0.5 * np.sqrt(1.0 + r[:, a, a] - r[:, b, b] - r[:, cc, cc])
            f = 0.25 / v
            xyz = np.empty((r.shape[0], 3))
            xyz[:, a] = v
            xyz[:, b] = (r[:, b, a] + r[:, a, b]) * f
            xyz[:, cc] = (r[:, cc, a] + r[:, a, cc]) * f
            q[sel] = np.concatenate([((r[:, cc, b] - r[:, b, cc]) * f)[:, None], xyz], axis=1)
    return q


def cutout_to_local(transform, basis_override) -> np.ndarray:
    """A cutout volume's Godot Transform3D T (matrix form: a point q of the unit shape, in the volume's own Godot axes -> its Godot
    position) -> the (3, 4) float32 [A | t] of gsr_cutout.to_local (a tested position -> q).  A Godot position p sits at F B p in frame
    space (F = diag(-1, -1, 1), B = basis_override: the convention of godot_to_frame), so to_local = (F B T)^-1.  It is composed and
    inverted in float64 and narrowed to float32 once.  With B a signed permutation (the identity, the usual PLY up-axis flips) this is
    also (F B T B^-1 F)^-1, the instance convention, since F B maps the unit cube and sphere onto themselves.  A singular transform
    raises LinAlgError."""
    T = np.asarray(transform, dtype=np.float64)
    if T.shape == (4, 4):
        T = T[:3]
    assert T.shape == (3, 4), T.shape
    Fb = np.eye(4)
    Fb[:3, :3] = np.diag([-1.0, -1.0, 1.0]) @ np.asarray(basis_override, dtype=np.float64).T
    M = np.eye(4)
    M[:3] = T
    return np.linalg.inv(Fb @ M)[:3].astype(np.float32)


def sort_pairs(keys: np.ndarray, values: np.ndarray | None = None, device: int = 0):
    """Host convenience around gsr_sort_pairs_host (stable LSD radix sort on the GPU)."""
    k = np.array(keys, dtype=np.uint32, copy=True)
    v = None if values is None else np.array(values, dtype=np.uint32, copy=True)
    u32p = C.POINTER(C.c_uint32)
    _lib.check(_lib.lib().gsr_sort_pairs_host(device, k.ctypes.data_as(u32p), None if v is None else v.ctypes.data_as(u32p),
                                              k.size), "gsr_sort_pairs_host")
    return (k, v) if v is not None else k
