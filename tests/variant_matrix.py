"""The variant matrix: one case per projection_kernel<INSTANCED, SH_BANDS, ORTHO, AA, DEPTH, CUT, HALF> instantiation, with the settings
that select no projection kernel spread over the cases by a covering design, and the composed reference frame of every case.

TEST INFRASTRUCTURE, shared by tests/test_variant_matrix.py (the kernels in the CPU emulator) and tests/test_gpu_variant_matrix.py (the
library through the C-ABI).  A case's reference frame is composed from the unchanged per-feature references:
  * the cloud a frame draws: the coefficients above the rendered degree set to zero (tests/test_sh_degree.zero_splat_coeffs), rounded to
    binary16 once for a binary16 store (tests/test_sh_half.rounded);
  * instanced frames: tests/instance_appearance_reference.frame (the default appearance for cases without one); frames without
    instances: tests/cutout_reference.oracle_frame (an empty set draws everything).  Both project with the instance, orthographic and
    anti-aliasing references, cut, sort (by view depth for the depth order) and composite (with the depth-compositing oracle when on);
  * motion: tests/motion_reference.splat_motion of the reference's records, then render_motion, with instance_prev_positions for
    instanced frames.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass

import numpy as np

from godotgaussiansplatting_b200.ply_file import swizzle_splats
from godotgaussiansplatting_b200.synthetic import synthetic_ply_table
from oracle import oracle as orc
from tests import cutout_reference as cr
from tests import instance_appearance_reference as ar
from tests import instance_reference as iref
from tests import motion_reference as mref
from tests import ortho_reference as oref
from tests.scenes import make_scene
from tests.test_instances import SCALED, rigid, rotation
from tests.test_sh_degree import zero_splat_coeffs
from tests.test_sh_half import rounded

F32, U32 = np.float32, np.uint32

# ---- the table -----------------------------------------------------------------------------------------------------------------
# the projection axes, in the order of projection_kernel's template parameters
AXES = ("inst", "bands", "ortho", "aa", "dord", "cut", "half")
AXIS_VALUES = {"inst": (False, True), "bands": (1, 2, 3, 4), "ortho": (False, True), "aa": (False, True), "dord": (False, True),
               "cut": (False, True), "half": (False, True)}
# composite_kernel<CONTRACT, DEPTH, MOTION>: (depth, motion) x contracted
COMPOSITORS = ("plain", "depth", "motion")
# the settings that select no projection kernel, with their values; `store`, `scene` and `appearance` only apply where noted
SETTINGS = {
    "compositor": tuple(itertools.product(COMPOSITORS, (True, False))),   # (variant, contract)
    "store": ("bands", "reduced"),      # a store of B bands, or a 4-band store rendered at degree B - 1 (B < 4 only)
    "heat": (False, True),
    "load_in": (False, True),           # time = 10 (static) or 0.6 (the load-in animation)
    "ragged": (False, True),            # a frame of whole 16 x 16 tiles, or a ragged one (each test file picks the two sizes)
    "scene": ("none", "plane"),         # depth and motion compositors only: no scene depth, or a plane over the right half
    "appearance": ("none", "mixed"),    # instanced cases only
}
AA_MOST, AA_SOME = 0.3, 0.1


def applies(setting: str, value, case) -> bool:
    """Can `setting` take `value` in a case with these projection axes and this compositor?"""
    if setting == "store" and value == "reduced":
        return case.bands < 4
    if setting == "scene":
        return case.compositor != "plain" or value == "none"
    if setting == "appearance":
        return case.inst or value == "none"
    return True


@dataclass(frozen=True)
class Case:
    inst: bool
    bands: int
    ortho: bool
    aa: bool
    dord: bool
    cut: bool
    half: bool
    compositor: str = "plain"
    contract: bool = True
    store: str = "bands"
    heat: bool = False
    load_in: bool = False
    ragged: bool = False
    scene: str = "none"
    appearance: str = "none"
    v: float = 0.0

    @property
    def id(self) -> str:
        on = [n for n, f in (("ortho", self.ortho), ("aa", self.aa), ("dord", self.dord), ("cut", self.cut), ("half", self.half)) if f]
        return "-".join(["inst" if self.inst else "flat", f"b{self.bands}"] + on)

    @property
    def kernel(self) -> tuple:
        """The projection_kernel template tuple (INSTANCED, SH_BANDS, ORTHO, AA, DEPTH, CUT, HALF) the case selects."""
        return tuple(getattr(self, a) for a in AXES)

    @property
    def compositor_kernel(self) -> tuple:
        """The composite_kernel template tuple (CONTRACT, DEPTH, MOTION)."""
        return (self.contract, self.compositor != "plain", self.compositor == "motion")

    @property
    def store_bands(self) -> int:
        return 4 if self.store == "reduced" else self.bands

    def setting(self, name):
        return (self.compositor, self.contract) if name == "compositor" else getattr(self, name)


def _spread(cases, setting, seed):
    """Each value of `setting` on about the same number of the cases where it applies: the admissible values dealt round-robin over a
    fixed pseudo-random order of the cases that admit them."""
    rng = np.random.default_rng(seed)
    groups = {}
    for c in cases:
        groups.setdefault(tuple(v for v in SETTINGS[setting] if applies(setting, v, c)), []).append(c)
    pick = {}
    for vals, cs in groups.items():
        order = rng.permutation(len(cs))
        for j, i in enumerate(order):
            pick[cs[i]] = vals[j % len(vals)]
    return pick


def _table():
    base = [Case(*t) for t in itertools.product(*(AXIS_VALUES[a] for a in AXES))]
    comp = _spread(base, "compositor", 1)
    rows = [Case(*c.kernel, compositor=comp[c][0], contract=comp[c][1]) for c in base]
    picks = {s: _spread(rows, s, seed) for seed, s in enumerate(("store", "heat", "load_in", "ragged", "scene", "appearance"), start=2)}
    out = []
    n_aa = 0
    for r in rows:
        v = 0.0
        if r.aa:
            v = AA_SOME if n_aa % 4 == 3 else AA_MOST   # 0.3 on most anti-aliased cases, 0.1 on every fourth
            n_aa += 1
        out.append(Case(*r.kernel, compositor=r.compositor, contract=r.contract, store=picks["store"][r], heat=picks["heat"][r],
                        load_in=picks["load_in"][r], ragged=picks["ragged"][r], scene=picks["scene"][r],
                        appearance=picks["appearance"][r], v=v))
    return out


CASES = _table()
IDS = [c.id for c in CASES]


def coverage_gaps(cases=CASES):
    """(setting, value, axis, axis value) pairs the table never puts together although a case could."""
    gaps = []
    for setting, values in SETTINGS.items():
        for value in values:
            for axis in AXES:
                for av in AXIS_VALUES[axis]:
                    possible = [c for c in cases if getattr(c, axis) == av and applies(setting, value, c)]
                    if not possible:
                        continue
                    if value not in {c.setting(setting) for c in possible}:
                        gaps.append((setting, value, axis, av))
    return gaps


# ---- the fixtures --------------------------------------------------------------------------------------------------------------
def cloud(n, seed=3):
    """A synthetic cloud with every SH coefficient non-zero."""
    t62 = synthetic_ply_table(n, seed)
    t62[:, 55:58] += 0.5
    t62[:, 9:54] += 0.02   # every coefficient non-zero
    return swizzle_splats(t62, 0.0)


def straddle(splat60, vp, w, h):
    """The cloud in the order of the camera's right axis, moved along it until the median splat centre projects onto the frame's left
    edge.  The frame's edge then runs through the projection warps of the middle ids: warps before them see no splat, warps after them
    many (the bulk SH copy), and the warps at the edge and at the rims of the cutout volumes few (the per-lane gather)."""
    V = np.asarray(vp, dtype=np.float64)[:16]
    right = np.array([V[0], V[4], V[8]]) / np.linalg.norm([V[0], V[4], V[8]])
    splat60 = splat60[np.argsort(splat60[:, 0:3].astype(np.float64) @ right, kind="stable")]
    p = splat60[:, 0:3].astype(np.float64)

    def median_x(k):
        q = (p + k * right).astype(F32)
        x, _, _ = mref.pix(vp, q[:, 0], q[:, 1], q[:, 2], w, h)
        return np.median(x)

    lo, hi = -20.0, 20.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if median_x(mid) < 0 else (lo, mid)
    out = splat60.copy()
    out[:, 0:3] = (p + lo * right).astype(F32)
    return out


def layout(n):
    """Four instances: a range ending at max_splats with an unaligned first (the clamped bulk copy), a source range drawn twice, and a
    scaled, non-rigid transform."""
    a, b = (2 * n) // 5, n // 2
    return [(0, a, rigid(4)), (a - n // 10, b, SCALED), (n - 301, 301, rigid(5)), (0, a, rigid(6))]


def previous_layout(inst):
    """The same ranges with other transforms: the previous frame of a motion case."""
    return [(f, c, rigid(40 + k, 0.3, 0.2)) for k, (f, c, _) in enumerate(inst)]


HIDDEN = ((1.0, 1.0, 1.0), 0.0, None)


def mixed_appearance(inst):
    """A tint above 1, opacity 0.5 with a draw count that is not a multiple of 32, the default, and a hidden instance."""
    draw = inst[1][1] // 3 + 1
    assert draw % 32 and draw < inst[1][1]
    return [((2.0, 0.5, 1.5), 1.0, None), ((1.0, 1.0, 1.0), 0.5, draw), ar.DEFAULT, HIDDEN]


def cutouts(splat60, fp):
    """A KEEP box in frame space and a REMOVE ellipsoid in source space, each around the bulk of the cloud."""
    sp = np.asarray(splat60, dtype=F32)[:, 0:3]
    fp = fp[np.isfinite(fp).all(1)]

    def vol(pts, frac, shape, action, space, axis, angle):
        c = np.median(pts, axis=0)
        h = np.median(np.abs(pts - c), axis=0) * frac + 1e-3
        A = np.diag(1.0 / h) @ rotation(axis, angle).T
        return cr.volume(np.concatenate([A, (-A @ c)[:, None]], axis=1), shape, action, space)

    return [vol(fp, 2.0, cr.BOX, cr.KEEP, cr.FRAME, [0.3, 1.0, 0.2], 0.3),
            vol(sp, 0.8, cr.ELLIPSOID, cr.REMOVE, cr.SOURCE, [1.0, -0.2, 0.5], -0.4)]


def camera(case, w, h, frame=25):
    """(vp, uniforms bytes) of the case's camera: the orbit camera at `frame`, orthographic or perspective, at the case's time."""
    if case.ortho:
        vp, ub = oref.ortho_camera(w, h, size=2.6, near=0.5, far=4.5, frame=frame)
    else:
        _, vp, ub = make_scene(16, 1, w, h, frame=frame)
    u = np.frombuffer(ub, dtype=F32).copy()
    u[6] = 0.6 if case.load_in else 10.0
    return np.ascontiguousarray(vp, dtype=F32), u.tobytes()


@dataclass
class Frame:
    """Everything a case draws: the inputs of the C-ABI calls and of the emulated kernels."""
    case: Case
    n: int
    w: int
    h: int
    splat60: np.ndarray      # the uploaded cloud
    src: np.ndarray          # the cloud the frame draws (zero-padded, and rounded for a binary16 store)
    vp: np.ndarray
    ub: bytes
    pvp: np.ndarray | None   # the previous frame of a motion case
    pub: bytes | None
    inst: list | None        # [(first, count, to_frame12)]
    prev_inst: list | None
    app: list | None
    vols: list | None
    Z: np.ndarray | None     # the scene depth

    @property
    def drawn(self):
        return iref.layout([(f, c) for f, c, _ in self.inst])[1] if self.inst else self.n


def frame_of(case, n, size, ragged_size):
    w, h = ragged_size if case.ragged else size
    vp, ub = camera(case, w, h)
    splat60 = straddle(cloud(n), vp, w, h)
    src = rounded(splat60, case.bands) if case.half else zero_splat_coeffs(splat60, case.bands)
    pvp = pub = None
    if case.compositor == "motion":
        pvp, pub = camera(case, w, h, frame=22)
    inst = prev_inst = app = None
    if case.inst:
        inst = layout(n)
        app = mixed_appearance(inst) if case.appearance == "mixed" else None
        if case.compositor == "motion":
            prev_inst = previous_layout(inst)
    vols = cutouts(splat60, cr.positions(splat60, 1.0, inst)[1]) if case.cut else None
    Z = None
    if case.scene == "plane":
        V = np.asarray(vp, dtype=np.float64)[:16].reshape(4, 4)
        d = -(splat60[:, 0:3].astype(np.float64) @ V[:3, 2] + V[3, 2])
        Z = np.full((h, w), np.inf, dtype=F32)
        Z[:, w // 2:] = np.median(d)
    return Frame(case, n, w, h, splat60, src, vp, ub, pvp, pub, inst, prev_inst, app, vols, Z)


def reference(fr: Frame) -> dict:
    """The composed reference frame of a case: every stage (tests/cutout_reference.oracle_frame's dict), and `motion` for motion cases."""
    c = fr.case
    depth = c.compositor != "plain"
    heat = 1.0 if c.heat else 0.0
    if c.inst:
        app = fr.app if fr.app is not None else [ar.DEFAULT] * len(fr.inst)
        ref = ar.frame(fr.src, fr.vp, fr.ub, fr.inst, app, c.v, c.ortho, fr.vols, heat, c.contract, fr.Z, depth, depth_order=c.dord)
    else:
        ref = cr.oracle_frame(fr.src, fr.vp, fr.ub, fr.vols if fr.vols is not None else [], c.v, c.ortho, heat, c.contract, None, fr.Z,
                              depth, depth_order=c.dord)
    ref["motion"] = None
    if c.compositor == "motion":
        prev_pos = None
        if c.inst:
            ranges = [(f, k) for f, k, _ in fr.inst]
            prev_pos = mref.instance_prev_positions(fr.src, ranges, [x for _, _, x in fr.prev_inst], 1.0, fr.drawn)
        m = mref.splat_motion(ref["records"], fr.vp, fr.pvp, fr.w, fr.h, prev_pos)
        rgba, dep, mo, staged = mref.render_motion(ref["records"], ref["values"], ref["bounds"], fr.w, fr.h, fr.vp, m, fr.Z, heat, c.contract)
        assert staged == ref["staged"]
        np.testing.assert_array_equal(bits(rgba), bits(ref["rgba"]))
        np.testing.assert_array_equal(bits(dep), bits(ref["depth"]))
        ref["motion"] = mo
    return ref


def bits(a):
    return np.ascontiguousarray(a).view(U32)


def warp_counts(values):
    """Emitting ids per warp of 32 drawn ids (the visible lanes of each projection warp)."""
    ids = np.unique(np.asarray(values, dtype=np.int64))
    return np.bincount(ids // 32)


def assert_both_phase2_paths(ref, bulk_min=12):
    """The frame has warps that take the bulk SH copy (>= bulk_min emitting lanes) and warps that gather per lane (1 .. bulk_min - 1)."""
    assert ref["m"] > 0 and ref["visible"] > 0
    wc = warp_counts(ref["unsorted_values"])
    assert (wc >= bulk_min).any(), "no warp takes the bulk SH copy"
    assert ((wc > 0) & (wc < bulk_min)).any(), "no warp gathers per lane"
