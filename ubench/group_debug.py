import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from tests.gsr_direct import Ctx
from tests.scenes import make_scene
from oracle import oracle as orc
def P(*a): print(time.strftime("%H:%M:%S"), *a, flush=True)
G = int(sys.argv[1]) if len(sys.argv) > 1 else 2
n, w, h = 30000, 640, 360
splat60, vp, ub = make_scene(n, 41, w, h, frame=0)
ctxs = [Ctx(n, w, h) for _ in range(G)]
P("created")
for c in ctxs: c.upload(splat60)
blobs = b"".join(c.group_export() for c in ctxs)
for r, c in enumerate(ctxs): c.group_attach(r, G, blobs)
P("attached")
for f in range(3):
    for r, c in enumerate(ctxs):
        c.render_async(vp, ub); P("frame", f, "enqueued rank", r)
    for r, c in enumerate(ctxs):
        try:
            c.sync(); P("frame", f, "synced rank", r, "M", c.stats().duplicates)
        except Exception as e:
            P("frame", f, "rank", r, "sync error:", e)
ref = orc.frame(splat60, vp, orc.uniforms_from_bytes(np.frombuffer(ub, dtype=np.uint8)))
gx = (w + 15) // 16
rows = (ref.keys >> 16) // gx
for r, c in enumerate(ctxs):
    t = c.taps(); sel = rows % G == r
    P("rank", r, "keys equal", np.array_equal(t["keys"], ref.keys[sel]), "values equal", np.array_equal(t["values"], ref.values[sel]), len(t["keys"]), int(sel.sum()))
img = ctxs[0].copy(6, w*h*4, np.float32).reshape(h, w, 4)
P("frame bit-identical", np.array_equal(img.view(np.uint32), ref.rgba.view(np.uint32)))
