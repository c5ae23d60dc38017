#!/bin/bash
# compute-sanitizer passes over a small but queue-exercising workload: 256x256 x 12 cascades, 3 updates + 5 fused frames, then
# the map query, the sea-state reduction and 4096 drifters reading a 256x256 wake layer.
cat > /tmp/san.py <<'PY'
import sys, numpy as np
sys.path.insert(0, ".")
import godotoceanwaves_b200 as gow
from bench import synth_params
g = gow.WaveGenerator(); g.map_size = 256; g.init_gpu(12)
p = [synth_params(gow.WaveCascadeParameters, c) for c in range(12)]
for _ in range(3):
    g.update_all(0.02, p)
g.update_frames(0.02, p, 5)        # fused frames: alternating scratch halves, column pass waiting for the previous frame's
d, n = g.maps_to_host()
pts = np.random.default_rng(0).uniform(-100, 100, (4096, 2)).astype(np.float32)
sc = gow.WaveGenerator.map_scales(p)
g.sample(pts, sc)
total, _ = g.sea_state(sc)                        # the sea-state reduction over every cascade
g.wake_init(256, 0.5)                             # drifters on the wake: the drift kernel's wake form
src = np.zeros(4, gow.WaveGenerator.WAKE_SOURCE)
src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = 20.0, 30.0, 3.0, 2.0, 0.2, -1
g.wake_step(0.05, 4, (0, 0), src)
dr = np.zeros(len(pts), gow.WaveGenerator.DRIFTER)
dr["x"], dr["z"], dr["scale"], dr["tilt"] = pts[:, 0], pts[:, 1], 1.0, 0.5
dp = gow.WaveGenerator.drift_params(current=(0.1, 0.0), box=(-100.0, -100.0, 200.0, 200.0), read_wake=True)
dr, inst = g.drift(dr, 1.0 / 60.0, sc, dp)
hv = np.array([[0, 0, 0], [2, 0, 0], [0, 1, 0], [0, 0, 1.5]], np.float32) - 0.4      # hull meshes: a shared tetrahedron
ht = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], np.int32)
hm = np.array([(0, 4, 0, 4, 1.0, 0.05)], gow.WaveGenerator.HULL_MESH)
g.set_hull_meshes(hm, hv, ht)
hb = np.zeros(256, gow.WaveGenerator.FLOATING_HULL)
hb["mass"], hb["inertia"] = 200.0, 50.0
hs = np.zeros(256, gow.WaveGenerator.BODY_STATE)
hs["position"][:, [0, 2]], hs["orientation"][:, 3] = pts[:256], 1.0
hs = g.simulate_hull_bodies(hb, hs, sc, 1.0 / 60.0, 4)
print("sea state", float(total["significant_wave_height"]), "drift", float(np.nansum(inst)), "hulls", float(np.nansum(hs["position"])))
print("checksum", int(d.view(np.uint16).astype(np.uint64).sum()), int(n.view(np.uint16).astype(np.uint64).sum()))
g.free()
PY
for tool in memcheck racecheck synccheck; do
  echo "== $tool"; timeout 600 compute-sanitizer --tool $tool python /tmp/san.py 2>&1 | grep -i "checksum\|sea state\|ERROR SUMMARY\|hazard\|error" | head -8
done
