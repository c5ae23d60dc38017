"""The floating-body ops as one application drives them, and the hull reduce at its edges.

Part 1: one generator takes a seeded plan of about 60 mixed calls -- every body op (ocean_buoyancy, ocean_body_forces,
ocean_simulate_bodies, ocean_simulate_driven_bodies, ocean_hull_forces, ocean_simulate_hull_bodies) and the surface query and
ray cast, in host and device form -- with body and point counts that grow and shrink, same-count calls on new contents,
caller and library outputs, mesh sets registered, rejected and released, the wake coupling switched on and off, and invalid
calls in between.  These calls share the generator's scratch (arrays that keep a larger call's data past a smaller call's
length), and every result must be byte-identical to the specification on maps copied to the host once.  Some calls are
repeated on a fresh generator, which must give the same bytes.  The plan's coverage is checked on the CPU.

Part 2: on maps made from a zero spectrum the water height is exactly +0, so with an identity rotation and t.y = 0 a vertex's
depth is exactly -y.  Triangles with corners at depths 0, subnormal and 1e-30 in every clip case, rotation and winding;
degenerate meshes; triangle and vertex counts around the 32-lane loop; body counts around the 8-bodies-per-block grid; depths
near the binary32 limit; and the integrator's accepted range -- ocean_hull_forces and ocean_simulate_hull_bodies against
oracle/hull.py byte for byte."""
import numpy as np
import pytest

from oracle import bodies as ob
from oracle import buoyancy as bu
from oracle import drag as dr
from oracle import drive as od
from oracle import hull as oh
from oracle import raycast as rc
from oracle import surface as su
from oracle import wake as wk
from oracle import wake_coupling as wc
from test_gpu_bodies import _bodies as _point_bodies
from test_gpu_drive import _drive
from test_gpu_hull import _bodies as _hull_bodies
from test_gpu_hull import _mesh_set
from test_gpu_wake_coupling import _flat, _init, _params, _same

N, C = 256, 3
RHO = 1025.0
DT = 1.0 / 60.0
TOL = 1e-3
INVALID = 1                                                     # OCEAN_ERR_INVALID_ARGUMENT
RAY_STEP, RAY_SAMPLES = 0.5, 128
WAKE_N, WAKE_DX = 128, 0.5                                      # the wake window spans [0, 64) m in x and z

# ---- the plan ------------------------------------------------------------------------------------------------------

OPS = ("query_surface", "raycast", "buoyancy", "body_forces", "simulate_bodies", "drive_bodies", "hull_forces", "simulate_hull_bodies")
SIMULATE = ("simulate_bodies", "drive_bodies", "simulate_hull_bodies")
HULL = ("hull_forces", "simulate_hull_bodies")
OPTIONAL_OUTPUTS = ("buoyancy", "body_forces", "hull_forces") + SIMULATE


def _op(op, form, n, seed, **kw):
    """One call: op in OPS, form host, device or both (host, then device on the same inputs), n bodies (points or rays for the
    query ops), seed of its scene.  Options: out (outputs given, else NULL), S (substeps), maxit, C (cascades), pts (range of
    points per body), zero (no world points), fleet (bodies and states kept across that fleet's calls), drive (full, thrusters
    or none), per (actuators per body), bad (NaN actuators), only (mesh indices), window (inside the wake window), replay."""
    step = dict(kind="op", op=op, form=form, n=n, seed=seed, out=True, S=1, maxit=8, C=C, pts=(1, 40), zero=False, fleet=None,
                drive="full", per=2, bad=False, only=None, window=False, replay=False)
    step.update(kw)
    return step


def _plan():
    """The seeded call sequence of test_mixed_sequence; deterministic."""
    P = [dict(kind="meshes", set="initial")]
    add = P.append
    add(_op("query_surface", "host", 3000, 1))
    add(_op("query_surface", "device", 3000, 2, C=2))
    add(_op("raycast", "host", 64, 3))
    add(_op("raycast", "device", 64, 4, replay=True))
    add(_op("buoyancy", "host", 200, 5, pts=(0, 200), out=True))           # ~2e4 world points
    add(_op("buoyancy", "device", 7, 6, out=False))
    add(_op("buoyancy", "device", 7, 7, out=True))
    add(_op("body_forces", "both", 33, 8, out=False, maxit=0))
    add(_op("body_forces", "host", 33, 9, out=True, replay=True))
    add(_op("simulate_bodies", "device", 1, 10, zero=True, out=True))
    add(_op("body_forces", "device", 9, 11, out=False, C=2))
    add(_op("hull_forces", "host", 200, 12, out=True))
    add(_op("hull_forces", "device", 9, 13, out=False))
    add(_op("hull_forces", "device", 9, 14, out=True))
    add(dict(kind="invalid", what="mesh"))
    add(_op("hull_forces", "host", 8, 15, out=False, replay=True))
    add(_op("simulate_bodies", "device", 33, 16, fleet="P", S=2, out=True))
    add(_op("simulate_bodies", "device", 33, 16, fleet="P", S=1, out=False))
    add(_op("simulate_bodies", "device", 33, 16, fleet="P", S=3, out=True))
    add(_op("simulate_bodies", "host", 9, 17, S=3, out=False))
    add(_op("simulate_bodies", "host", 9, 18, S=1, out=True, replay=True))
    add(dict(kind="invalid", what="substeps"))
    add(_op("drive_bodies", "host", 200, 19, per=3, out=True))
    add(_op("drive_bodies", "device", 8, 20, fleet="D", per=2, out=False))
    add(_op("drive_bodies", "device", 8, 20, fleet="D", drive="none", out=True))    # after tethers: the plain integrator, a zero record
    add(_op("drive_bodies", "device", 8, 20, fleet="D", drive="thrusters", per=1, out=True))
    add(_op("drive_bodies", "host", 8, 21, drive="none", out=False))
    add(_op("drive_bodies", "host", 8, 22, drive="thrusters", per=3, out=True, replay=True))
    add(_op("drive_bodies", "both", 33, 23, per=1, bad=True, out=True, S=2))
    add(_op("simulate_hull_bodies", "device", 7, 24, fleet="H", S=2, out=True))
    add(_op("simulate_hull_bodies", "device", 7, 24, fleet="H", S=1, out=False))
    add(_op("simulate_hull_bodies", "host", 33, 25, out=False, S=2))
    add(_op("simulate_hull_bodies", "host", 33, 26, out=True, replay=True))
    add(dict(kind="meshes", set="large"))
    add(_op("hull_forces", "host", 9, 27, only=[11], out=True, replay=True))    # 9 bodies on the 2112-vertex hull
    add(_op("simulate_hull_bodies", "both", 33, 28, S=2, out=True))
    add(dict(kind="meshes", set="rejected"))                                      # the large set stays live
    add(_op("hull_forces", "device", 17, 29, out=False))
    add(dict(kind="meshes", set="small"))
    add(_op("hull_forces", "host", 1, 30, out=True))
    add(_op("simulate_hull_bodies", "host", 8, 31, out=True, S=1, replay=True))
    add(dict(kind="wake", what="on"))
    add(_op("query_surface", "host", 600, 32, window=True))
    add(_op("buoyancy", "host", 9, 33, window=True, out=True))
    add(_op("body_forces", "device", 9, 34, window=True, out=True))
    add(_op("simulate_bodies", "host", 8, 35, window=True, S=2, out=True))
    add(_op("drive_bodies", "device", 9, 36, window=True, per=2, out=True))
    add(_op("hull_forces", "host", 7, 37, window=True, out=True))
    add(_op("simulate_hull_bodies", "device", 7, 38, window=True, S=2, out=True))
    add(dict(kind="wake", what="step"))
    add(_op("hull_forces", "device", 7, 39, window=True, out=True))
    add(_op("raycast", "host", 40, 40, window=True))
    add(dict(kind="invalid", what="density"))
    add(_op("body_forces", "host", 7, 41, window=True, out=True))
    add(dict(kind="wake", what="off"))
    add(_op("body_forces", "host", 7, 42, out=True))
    add(dict(kind="meshes", set="empty"))
    add(dict(kind="invalid", what="empty"))
    add(_op("buoyancy", "host", 1, 43, out=False, replay=True))
    add(dict(kind="meshes", set="again"))
    add(_op("hull_forces", "host", 33, 44, out=True, replay=True))
    add(_op("hull_forces", "host", 33, 45, out=False))
    add(_op("simulate_hull_bodies", "device", 9, 46, out=False, S=3))
    add(_op("simulate_hull_bodies", "device", 9, 47, out=True, S=1))
    add(_op("simulate_bodies", "device", 7, 48, out=True, S=1))
    add(_op("simulate_bodies", "device", 7, 49, out=False, S=2, C=2))
    add(_op("buoyancy", "both", 33, 50, out=True))
    add(_op("raycast", "device", 40, 51))
    add(_op("query_surface", "device", 1, 52, replay=True))
    add(_op("drive_bodies", "device", 7, 53, per=1, out=True))
    add(_op("drive_bodies", "device", 7, 54, per=2, out=False))
    return P


def _mesh_sets():
    """The mesh sets the plan registers: initial (_mesh_set's 8 meshes), large (11 meshes, the last a 2112-vertex sphere),
    small (a box and an empty mesh), rejected (the large set with a negative drag coefficient), empty; again is initial."""
    initial = _mesh_set(np.random.default_rng(101), 5)
    m, v, t = _mesh_set(np.random.default_rng(102), 8)
    nu, nv = 64, 32
    th = np.linspace(0, np.pi, nv + 1)
    ph = np.linspace(0, 2 * np.pi, nu, endpoint=False)
    grid = np.stack([np.outer(np.sin(th), np.cos(ph)), np.outer(np.cos(th), np.ones(nu)), np.outer(np.sin(th), np.sin(ph))], 2)
    sv = (grid.reshape(-1, 3) * (4.0, 1.5, 2.5)).astype(np.float32)
    idx = np.arange((nv + 1) * nu).reshape(nv + 1, nu)
    a, b = idx[:-1], np.roll(idx[:-1], -1, 1)
    c, d = idx[1:], np.roll(idx[1:], -1, 1)
    st = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)]).astype(np.int32)
    sphere = np.array([(len(v), len(sv), len(t), len(st), 1.0, 0.05)], oh.MESH)
    large = (np.concatenate([m, sphere]), np.concatenate([v, sv]), np.concatenate([t, st]))
    assert len(large[0]) == 12 and large[0]["num_vertices"][11] == len(sv) == 2112
    small = (initial[0][[6, 7]].copy(), initial[1], initial[2])
    rejected = (large[0].copy(), large[1], large[2])
    rejected[0]["tangential_drag"][3] = -1.0
    empty = (np.zeros(0, oh.MESH), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    return dict(initial=initial, large=large, small=small, rejected=rejected, empty=empty, again=initial)


def _window(rng, n):
    return rng.uniform(5.0, 60.0, (n, 2))


def _inputs(step, meshes):
    """The arguments of an op step (fleet steps: the fleet's bodies and first states), from its seed and the live mesh set."""
    seed = step["seed"]
    rng = np.random.default_rng(1000 + seed)
    n, op = step["n"], step["op"]
    if op == "query_surface":
        pts = _window(rng, n) if step["window"] else rng.uniform(-150.0, 150.0, (n, 2))
        return dict(points=pts.astype(np.float32))
    if op == "raycast":
        r = np.zeros(n, rc.RAY)
        xz = _window(rng, n) if step["window"] else rng.uniform(-100.0, 100.0, (n, 2))
        oy = rng.uniform(-4.0, 6.0, n)
        r["origin"] = np.stack([xz[:, 0], oy, xz[:, 1]], 1)
        d = rng.normal(size=(n, 3))
        d[:, 1] = -np.sign(oy) * np.abs(d[:, 1]) - 0.1
        r["direction"] = d / np.linalg.norm(d, axis=1, keepdims=True)
        r["t_max"] = rng.uniform(5.0, 25.0, n)
        return dict(rays=r)
    if op in HULL:
        ms = meshes[0]
        fb, s = _hull_bodies(rng, n, ms, span=40.0)
        if step["only"] is not None:
            fb["mesh"] = rng.choice(step["only"], n)
        if step["window"]:
            s["position"][:, [0, 2]] = _window(rng, n)
        table, vel = oh.pose(fb, s)
        return dict(bodies=fb, states=s, table=table, vel=vel, world=int(ms["num_vertices"].astype(np.int64)[fb["mesh"]].sum()))
    lo, hi = step["pts"]
    sizes = np.random.default_rng(2000 + seed).integers(max(lo, 1), hi + 1, n)
    b, s, hull, cda = _point_bodies(3000 + seed, sizes)
    if step["zero"]:
        b["num_points"] = 0
    elif lo == 0:
        b["num_points"][::5] = 0
    if step["window"]:
        s["position"][:, [0, 2]] = _window(rng, n)
    table, vel = ob.pose(b, s)
    args = dict(bodies=b, states=s, hull=hull, cda=cda, table=table, vel=vel, world=int(b["num_points"].astype(np.int64).sum()))
    if op == "drive_bodies":
        th, fo, ld, te, _ = _drive(rng, s, step["per"], bad=step["bad"])
        if step["drive"] == "none":
            th, fo, ld, te = th[:0], fo[:0], None, te[:0]
        elif step["drive"] == "thrusters":
            fo, ld, te = fo[:0], None, te[:0]
        args.update(thrusters=th, foils=fo, loads=ld, tethers=te)
    return args


def _needs(step, args):
    """Elements of each shared array a call needs, from its arguments: the host path grows every array it uses to at least
    this, and a later smaller call finds the earlier call's data past its own length."""
    op, B, out = step["op"], step["n"], step["out"]
    need = {}
    if op in ("query_surface", "raycast"):
        return {"query": B} if op == "query_surface" else {}
    world = args["world"]
    if op in HULL:
        need.update(hull_poses=B, velocities=B, offsets=B, q=world, corners=2 * world, query=world)
        if op == "hull_forces" and not out:
            need["samples"] = world
    else:
        need.update(poses=B, offsets=B, q=world, query=world)
        if op != "buoyancy":
            need["velocities"] = B
        if op in ("buoyancy", "body_forces") and not out:
            need["samples"] = world
    if op in SIMULATE:
        need.update(r2=B, rows=B, samples=need["q"])
        if op == "simulate_hull_bodies":
            need["hull_rows"] = B
        if not out:
            need.update(hydrostatic=B, drag=B)
    if op == "drive_bodies":
        nt, nf, nte = len(args["thrusters"]), len(args["foils"]), len(args["tethers"])
        if nt or nf or nte or args["loads"] is not None:
            for k in ("q", "samples", "query"):
                need[k] += nt + nf
            ends = int((args["tethers"]["body_b"] >= 0).sum())
            need.update(thrusters=nt, foils=nf, tethers=nte, tether_forces=nte, sums=B, incidence=B + 1 + nt + nf + nte + ends)
            if args["loads"] is not None:
                need["loads"] = B
            if not out:
                need.update(drive=B, tensions=nte)
    return {k: v for k, v in need.items() if v > 0}


def _walk(plan):
    """Each op step with its arguments and needs, the live mesh set and the coupling state: [(index, step, args, needs, wake)]."""
    sets = _mesh_sets()
    live, wake, out = None, False, []
    for i, step in enumerate(plan):
        if step["kind"] == "meshes":
            if step["set"] != "rejected":
                live = sets[step["set"]] if step["set"] != "empty" else None
        elif step["kind"] == "wake":
            wake = step["what"] != "off"
        elif step["kind"] == "op":
            args = _inputs(step, live)
            out.append((i, step, args, _needs(step, args), wake))
    return out


SHARED = ("poses", "hull_poses", "velocities", "offsets", "r2", "rows", "hull_rows", "q", "samples", "corners", "hydrostatic", "drag",
          "thrusters", "foils", "loads", "tethers", "tether_forces", "incidence", "sums", "drive", "tensions", "query")


def test_plan_covers_the_sequence():
    """The plan reaches every op in both forms, leaves every shared array larger than the next call that uses it needs, calls
    every op twice in a row at one count on new contents, gives and leaves out the optional outputs in both orders, walks the
    mesh set through every transition and runs ops with the coupling on and off."""
    plan = _plan()
    walk = _walk(plan)
    assert 55 <= len(walk) <= 70
    forms = {(s["op"], f) for _, s, _, _, _ in walk for f in (("host", "device") if s["form"] == "both" else (s["form"],))}
    assert forms == {(op, f) for op in OPS for f in ("host", "device")}
    assert {1, 7, 8, 9, 33, 200} <= {s["n"] for _, s, _, _, _ in walk if s["op"] not in ("query_surface", "raycast")}
    worlds = [n["q"] if "q" in n else 0 for _, s, _, n, _ in walk if s["op"] not in ("query_surface", "raycast")]
    assert min(worlds) == 0 and max(worlds) >= 10000
    # every shared array: the previous call that used it needed more than the next one does
    for name in SHARED:
        users = [n[name] for _, _, _, n, _ in walk if name in n]
        assert any(a > b for a, b in zip(users, users[1:])), name
    # same count, new contents, back to back, for every op
    pairs = set()
    for (_, a, x, _, _), (_, b, y, _, _) in zip(walk, walk[1:]):
        if a["op"] == b["op"] and a["n"] == b["n"] and a["fleet"] is None and b["fleet"] is None:
            keys = [k for k in x if k in ("points", "rays", "bodies", "states")]
            if all(x[k].tobytes() != y[k].tobytes() for k in keys):
                pairs.add(a["op"])
    assert pairs == set(OPS)
    # outputs given then left out, and left out then given
    for op in OPTIONAL_OUTPUTS:
        outs = [s["out"] for _, s, _, _, _ in walk if s["op"] == op]
        assert (True, False) in zip(outs, outs[1:]) and (False, True) in zip(outs, outs[1:]), op
    # device fleets advance one state tensor over consecutive calls
    for fleet in ("P", "D", "H"):
        assert sum(s["fleet"] == fleet for _, s, _, _, _ in walk) >= 2
    # a driven call without drive rows right after one with tethers
    drives = [(s, a) for _, s, a, _, _ in walk if s["op"] == "drive_bodies"]
    assert any(len(a["tethers"]) and s2["drive"] == "none" for (s, a), (s2, _) in zip(drives, drives[1:]))
    assert len({len(a["thrusters"]) + len(a["foils"]) for _, a in drives}) >= 4
    # the mesh set: larger, smaller, rejected, released, registered again; hull calls under every live set
    sets = _mesh_sets()
    seq = [s["set"] for s in plan if s["kind"] == "meshes"]
    assert seq == ["initial", "large", "rejected", "small", "empty", "again"]
    assert len(sets["large"][0]) > len(sets["initial"][0]) > len(sets["small"][0])
    assert len(sets["large"][1]) > len(sets["initial"][1]) and len(sets["large"][2]) > len(sets["initial"][2])
    for a, b in zip(seq, seq[1:]):
        between = plan[plan.index(dict(kind="meshes", set=a)) + 1:plan.index(dict(kind="meshes", set=b))]
        assert any(s["kind"] in ("op", "invalid") and (s.get("op") in HULL or s.get("what") in ("mesh", "empty")) for s in between), a
    # the coupling on for part of the sequence, stepped while on, then off
    assert {w for *_, w in walk} == {False, True}
    wake = [s["what"] for s in plan if s["kind"] == "wake"]
    assert wake == ["on", "step", "off"]
    assert {s["op"] for _, s, _, _, w in walk if w} >= set(OPS) - {"raycast"}
    # invalid calls between valid ones, and replays on a fresh generator spread through the plan
    assert [s["what"] for s in plan if s["kind"] == "invalid"] == ["mesh", "substeps", "density", "empty"]
    replays = [i for i, s, _, _, w in walk if s["replay"]]
    assert 8 <= len(replays) <= 12 and not any(w for _, s, _, _, w in walk if s["replay"])
    assert replays[0] < len(plan) // 6 and replays[-1] > 5 * len(plan) // 6


# ---- running the plan --------------------------------------------------------------------------------------------------

def _dev(a):
    import torch
    b = np.ascontiguousarray(a).tobytes()
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if b else None


def _zeros(n, dtype):
    import torch
    return torch.zeros(max(n, 1) * np.dtype(dtype).itemsize, dtype=torch.uint8, device="cuda")


def _back(t, dtype, n):
    return np.frombuffer(t.cpu().numpy().tobytes(), dtype)[:n].copy()


def _ptr(t):
    return None if t is None else t.data_ptr()


class _Runner:
    """Runs op steps on a generator: the host or device form, returning the outputs in the specification's order."""

    def __init__(self, g, scales):
        from godotoceanwaves_b200.native import check, load_library
        self.g, self.scales, self.lib, self.check = g, scales, load_library(), check

    def host(self, step, a, states=None):
        g, c, S, mi, out = self.g, step["C"], step["S"], step["maxit"], step["out"]
        sc = self.scales[:c]
        op = step["op"]
        if op == "query_surface":
            return (g.query_surface(a["points"], sc, TOL, mi),)
        if op == "raycast":
            return (g.raycast(a["rays"], sc, RAY_STEP, RAY_SAMPLES, TOL, mi),)
        if op == "buoyancy":
            r = g.buoyancy(a["table"], a["hull"], sc, RHO, TOL, mi, return_samples=out)
            return r if out else (r,)
        if op == "body_forces":
            return g.body_forces(a["table"], a["vel"], a["hull"], a["cda"], sc, RHO, TOL, mi, return_samples=out)
        if op == "hull_forces":
            return g.hull_forces(a["table"], a["vel"], sc, RHO, TOL, mi, return_samples=out)
        if op == "simulate_bodies":
            r = g.simulate_bodies(a["bodies"], states, a["hull"], a["cda"], sc, DT, S, RHO, TOL, mi, return_records=out, return_transforms=out)
        elif op == "drive_bodies":
            r = g.drive_bodies(a["bodies"], states, a["hull"], a["cda"], sc, DT, S, RHO, TOL, mi, thrusters=a["thrusters"], foils=a["foils"],
                               loads=a["loads"], tethers=a["tethers"], return_records=out, return_tensions=out, return_transforms=out)
        else:
            r = g.simulate_hull_bodies(a["bodies"], states, sc, DT, S, RHO, TOL, mi, return_records=out, return_transforms=out)
        return r if out else (r,)

    def device(self, step, a, st_dev=None):
        """The _device form; simulate ops advance st_dev (a uint8 tensor of STATE rows) in place and return its new states."""
        import torch
        g, lib, c, S, mi, out = self.g, self.lib, step["C"], step["S"], step["maxit"], step["out"]
        sc = np.ascontiguousarray(self.scales[:c])
        op, n, ctx = step["op"], step["n"], g.context
        torch.cuda.synchronize()
        if op == "query_surface":
            o = _zeros(n, su.RECORD)
            self.check(lib.ocean_query_surface_device(ctx, n, _ptr(_dev(a["points"])), c, sc.ctypes.data, TOL, mi, o.data_ptr()))
            g.synchronize()
            return (_back(o, su.RECORD, n),)
        if op == "raycast":
            o = _zeros(n, rc.HIT)
            self.check(lib.ocean_raycast_device(ctx, n, _ptr(_dev(a["rays"])), c, sc.ctypes.data, RAY_STEP, RAY_SAMPLES, TOL, mi, o.data_ptr()))
            g.synchronize()
            return (_back(o, rc.HIT, n),)
        world = a["world"]
        if op not in HULL:
            P, pts, cda = len(a["hull"]), _dev(a["hull"]), _dev(a["cda"])
        smp = _zeros(world, su.RECORD) if out and op in ("buoyancy", "body_forces", "hull_forces") else None
        hyd = _zeros(n, bu.RESULT) if out or op in ("buoyancy", "body_forces", "hull_forces") else None
        drg = _zeros(n, dr.RESULT) if out or op in ("body_forces", "hull_forces") else None
        T = torch.zeros(n * 12, dtype=torch.float32, device="cuda") if out and op in SIMULATE else None
        if op == "buoyancy":
            self.check(lib.ocean_buoyancy_device(ctx, n, a["table"].ctypes.data, P, _ptr(pts), c, sc.ctypes.data, RHO, TOL, mi, hyd.data_ptr(),
                                                 _ptr(smp)))
            g.synchronize()
            return (_back(hyd, bu.RESULT, n),) + ((_back(smp, su.RECORD, world),) if out else ())
        if op == "body_forces":
            self.check(lib.ocean_body_forces_device(ctx, n, a["table"].ctypes.data, a["vel"].ctypes.data, P, _ptr(pts), _ptr(cda), c,
                                                    sc.ctypes.data, RHO, TOL, mi, hyd.data_ptr(), drg.data_ptr(), _ptr(smp)))
            g.synchronize()
            return (_back(hyd, bu.RESULT, n), _back(drg, dr.RESULT, n)) + ((_back(smp, su.RECORD, world),) if out else ())
        if op == "hull_forces":
            self.check(lib.ocean_hull_forces_device(ctx, n, a["table"].ctypes.data, a["vel"].ctypes.data, c, sc.ctypes.data, RHO, TOL, mi,
                                                    hyd.data_ptr(), drg.data_ptr(), _ptr(smp)))
            g.synchronize()
            return (_back(hyd, bu.RESULT, n), _back(drg, dr.RESULT, n)) + ((_back(smp, su.RECORD, world),) if out else ())
        fb = np.ascontiguousarray(a["bodies"])
        extra = ()
        if op == "simulate_bodies":
            self.check(lib.ocean_simulate_bodies_device(ctx, n, fb.ctypes.data, st_dev.data_ptr(), P, _ptr(pts), _ptr(cda), c, sc.ctypes.data,
                                                        RHO, DT, S, TOL, mi, _ptr(hyd), _ptr(drg), _ptr(T)))
        elif op == "drive_bodies":
            th, fo, ld, te = a["thrusters"], a["foils"], a["loads"], a["tethers"]
            drv = _zeros(n, od.RESULT) if out else None
            ten = torch.zeros(max(len(te), 1), dtype=torch.float32, device="cuda") if out else None
            hp = lambda x: x.ctypes.data if x is not None and len(x) else None  # noqa: E731
            self.check(lib.ocean_simulate_driven_bodies_device(
                ctx, n, fb.ctypes.data, st_dev.data_ptr(), P, _ptr(pts), _ptr(cda), c, sc.ctypes.data, RHO, DT, S, TOL, mi, len(th), hp(th),
                len(fo), hp(fo), hp(ld), len(te), hp(te), _ptr(hyd), _ptr(drg), _ptr(drv), _ptr(ten), _ptr(T)))
            if out:
                extra = (drv, ten, len(te))
        else:
            self.check(lib.ocean_simulate_hull_bodies_device(ctx, n, fb.ctypes.data, st_dev.data_ptr(), c, sc.ctypes.data, RHO, DT, S, TOL, mi,
                                                             _ptr(hyd), _ptr(drg), _ptr(T)))
        g.synchronize()
        s = _back(st_dev, ob.STATE, n)
        if not out:
            return (s,)
        res = (s, _back(hyd, bu.RESULT, n), _back(drg, dr.RESULT, n))
        if extra:
            res += (_back(extra[0], od.RESULT, n), extra[1].cpu().numpy()[:extra[2]].copy())
        return res + (T.cpu().numpy().reshape(n, 12).copy(),)


def _spec(step, a, states, maps, scales, meshes, cp):
    """The specification of an op step, in the order the runner returns, cut to the outputs the step asks for."""
    d16, n16, vel = (m[:step["C"]] for m in maps)
    sc, S, mi, op = scales[:step["C"]], step["S"], step["maxit"], step["op"]
    with np.errstate(all="ignore"):
        if op == "query_surface":
            return (wc.query_surface(d16, n16, a["points"], sc, TOL, mi, cp),)
        if op == "raycast":
            return (rc.raycast(d16, n16, a["rays"], sc, RAY_STEP, RAY_SAMPLES, TOL, mi),)
        if op == "buoyancy":
            r = wc.buoyancy(d16, n16, a["table"], a["hull"], sc, RHO, TOL, mi, True, cp)
            return r if step["out"] else r[:1]
        if op == "body_forces":
            r = wc.body_forces(d16, n16, vel, a["table"], a["vel"], a["hull"], a["cda"], sc, RHO, TOL, mi, True, cp)
        elif op == "hull_forces":
            r = oh.hull_forces(d16, n16, vel, a["table"], a["vel"], *meshes, sc, RHO, TOL, mi, True, wake=cp)
        elif op == "simulate_bodies":
            r = wc.simulate(d16, n16, vel, a["bodies"], states, a["hull"], a["cda"], sc, RHO, DT, S, TOL, mi, cp)
        elif op == "drive_bodies":
            r = od.simulate(d16, n16, vel, a["bodies"], states, a["hull"], a["cda"], sc, RHO, DT, S, TOL, mi, a["thrusters"], a["foils"], a["loads"],
                            a["tethers"], cp)
        else:
            r = oh.simulate(d16, n16, vel, a["bodies"], states, *meshes, sc, RHO, DT, S, TOL, mi, wake=cp)
    if op in ("body_forces", "hull_forces"):
        return r if step["out"] else r[:2]
    return r if step["out"] else r[:1]


def _assert_same(got, want, what):
    assert len(got) == len(want), what
    for k, (x, y) in enumerate(zip(got, want)):
        assert _same(x, y), f"{what}: output {k} differs from the specification"


def _identical(a, b, what):
    assert len(a) == len(b), what
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes(), f"{what}: output {k}"


def _fresh(meshes):
    """A new generator with the parameters and updates of the plan's, and the live mesh set."""
    from test_gpu_sampling import _gen
    _, g, _ = _gen(N, C)
    g.update_velocity()
    if meshes is not None:
        g.set_hull_meshes(*meshes)
    return g


@pytest.mark.gpu
def test_mixed_sequence():
    """The plan on one generator at N = 256, C = 3: every call byte-identical to its specification (a NaN only has to meet a
    NaN), host and device forms of one call identical, invalid calls rejected with no launch, hull calls refused while no set
    is registered, and about ten calls repeated on a fresh generator with the same bytes."""
    import torch

    from godotoceanwaves_b200.native import OceanError
    from test_gpu_sampling import _gen
    gow, g, params = _gen(N, C)
    scales = np.ascontiguousarray(gow.WaveGenerator.map_scales(params), np.float32)
    g.update_velocity()
    d16, n16 = g.maps_to_host(0, C)
    maps = (d16, n16, g.velocity_to_host(0, C))
    run = _Runner(g, scales)
    sets = _mesh_sets()
    live = None
    layer = cp = None
    fleets = {}
    src = np.zeros(3, wk.SOURCE)
    src["x"], src["z"], src["vx"], src["radius"], src["head"], src["body"] = (10.0, 20.0, 30.0), (15.0, 30.0, 40.0), 2.0, 3.0, 0.4, -1
    last = {}                                                   # the last valid inputs of each op, for the invalid calls
    replays = 0
    for i, step in enumerate(_plan()):
        kind = step["kind"]
        if kind == "meshes":
            m = sets[step["set"]]
            if step["set"] == "rejected":
                before = g.info().kernel_launches
                with pytest.raises(OceanError, match=f"status {INVALID}:"):
                    g.set_hull_meshes(*m)
                assert g.info().kernel_launches == before
                continue
            vols = g.set_hull_meshes(*m)
            np.testing.assert_allclose(vols, oh.volumes(*m), rtol=1e-6)
            live = m if step["set"] != "empty" else None
            continue
        if kind == "wake":
            if step["what"] == "on":
                p = _params(WAKE_N, WAKE_DX, damping=0.02, sponge_cells=16)
                _init(g, p)
                layer, cp = wk.Layer(p), wc.Coupling(WAKE_N, WAKE_DX)
                g.wake_set_coupling(True)
                steps = 2
            elif step["what"] == "step":
                steps = 1
            else:
                g.wake_set_coupling(False)
                cp = None
                continue
            for _ in range(steps):
                g.wake_step(DT, 2, (0, 0), src)
                wc.step(layer, cp, DT, 2, (0, 0), src, None)
            continue
        if kind == "invalid":
            before = g.info().kernel_launches
            sc = scales
            if step["what"] == "mesh":
                a = last["hull_forces"]
                bad = a["table"].copy()
                bad["mesh"][len(bad) // 2] = len(live[0])
                calls = [lambda: g.hull_forces(bad, a["vel"], sc, RHO)]
            elif step["what"] == "substeps":
                a = last["simulate_bodies"]
                d = last["drive_bodies"] if "drive_bodies" in last else a
                calls = [lambda: g.simulate_bodies(a["bodies"], a["states"], a["hull"], a["cda"], sc, DT, 65, RHO),
                         lambda: g.drive_bodies(a["bodies"], a["states"], a["hull"], a["cda"], sc, DT, 65, RHO, thrusters=d.get("thrusters"))]
            elif step["what"] == "density":
                a = last["buoyancy"]
                calls = [lambda: g.buoyancy(a["table"], a["hull"], sc, -1.0),
                         lambda: g.hull_forces(last["hull_forces"]["table"], last["hull_forces"]["vel"], sc, -1.0)]
            else:                                               # no mesh set: every hull call is refused
                h, s = last["hull_forces"], last["simulate_hull_bodies"]
                calls = [lambda: g.hull_forces(h["table"], h["vel"], sc, RHO),
                         lambda: g.simulate_hull_bodies(s["bodies"], s["states"], sc, DT, 1, RHO)]
            for call in calls:
                with pytest.raises(OceanError, match=f"status {INVALID}:"):
                    call()
            assert g.info().kernel_launches == before, step
            continue
        # an op step
        op = step["op"]
        what = f"step {i} ({op}, {step['form']}, n = {step['n']})"
        a = _inputs(step, live)
        states = None
        if step["fleet"] is not None:
            if step["fleet"] not in fleets:
                fleets[step["fleet"]] = dict(states=a["states"].copy(), dev=_dev(a["states"]))
            fl = fleets[step["fleet"]]
            states = fl["states"]
        elif op in SIMULATE:
            states = a["states"]
        want = _spec(step, a, states, maps, scales, live, cp)
        if step["form"] in ("host", "both"):
            got = run.host(step, a, states)
            _assert_same(got, want, what + " host")
        if step["form"] in ("device", "both"):
            st = fl["dev"] if step["fleet"] is not None else (_dev(states) if states is not None else None)
            dgot = run.device(step, a, st)
            _assert_same(dgot, want, what + " device")
            if step["form"] == "both":
                _identical(got, dgot, what + " host and device")
            got = dgot
        if step["fleet"] is not None:
            fl["states"] = want[0]
        last[op] = a
        if step["replay"]:
            replays += 1
            fresh = _fresh(live)
            try:
                _identical(_Runner(fresh, scales).host(step, a, states), got, what + " on a fresh generator")
            finally:
                fresh.free()
        torch.cuda.synchronize()
    assert replays >= 8
    g.free()


# ---- the hull reduce at its edges, on exactly flat maps ---------------------------------------------------------------

RHO_G = RHO * 9.81
TINY = (0.0, 2.0 ** -149, 1e-40, 1e-30)                         # 0, the smallest subnormal, a subnormal, a normal whose square underflows


def _clip_patterns():
    """Corner heights y (depth -y) per clip case, with one or two corners at +-e for each e of TINY: [(wet count, y0, y1, y2)]."""
    out = []
    for e in TINY:
        for z in ((e, -e) if e else (0.0,)):
            out += [(0, z, z, 1.0), (0, z, 1.0, 1.5), (1, -1.0, z, 1.0), (1, -1.0, z, z), (2, -1.0, -1.5, z), (2, z, -1.0, 0.5),
                    (3, -1.0, -2.0, -0.5), (3, -1.0, z, -2.0)]
    return out


def _clip_meshes():
    """One single-triangle mesh per pattern, corner rotation and winding: (MESH [M], vertices, triangles, heights [M][3])."""
    xz = np.array([[0.0, 0.0], [1.5, 0.25], [0.5, 1.25]])
    meshes, verts, tris, heights = [], [], [], []
    for _, *y in _clip_patterns():
        for rot in range(3):
            for wind in ((0, 1, 2), (0, 2, 1)):
                order = [(rot + k) % 3 for k in range(3)]
                v = np.array([[xz[k, 0], y[k], xz[k, 1]] for k in order], np.float32)
                meshes.append((3 * len(meshes), 3, len(meshes), 1, 1.1, 0.07))
                verts.append(v)
                tris.append(wind)
                heights.append(v[list(wind), 1])
    return np.array(meshes, oh.MESH), np.concatenate(verts), np.array(tris, np.int32), np.array(heights)


def _hand_force(p):
    """-rho g integral(d n dA) over the wet part (d = -y > 0) of the triangle p [3][3] (Godot's winding), in float64: the
    triangle clipped to y < 0 as a polygon, fanned from its first corner."""
    p = np.asarray(p, np.float64)
    poly = []
    for k in range(3):
        a, b = p[k], p[(k + 1) % 3]
        if a[1] < 0:
            poly.append(a)
        if (a[1] < 0) != (b[1] < 0) and a[1] != b[1]:
            t = a[1] / (a[1] - b[1])
            x = a + t * (b - a)
            x[1] = 0.0
            poly.append(x)
    f = np.zeros(3)
    for k in range(1, len(poly) - 1):
        c0, c1, c2 = poly[0], poly[k], poly[k + 1]
        area = 0.5 * np.cross(c2 - c0, c1 - c0)
        f += area * -(c0[1] + c1[1] + c2[1]) / 3.0
    return -RHO_G * f


def _identity(B, rng=None, ty=0.0):
    s = np.zeros(B, ob.STATE)
    s["orientation"] = (0, 0, 0, 1)
    s["position"][:, 1] = ty
    if rng is not None:
        s["position"][:, [0, 2]] = rng.uniform(-40.0, 40.0, (B, 2))
        s["linear_velocity"] = rng.normal(size=(B, 3))
        s["angular_velocity"] = rng.normal(size=(B, 3)) * 0.3
    return s


@pytest.fixture(scope="module")
def flat():
    """A 256^2 x 2 generator on flat maps, with those maps on the host: (generator, scales, (d16, n16, velocity))."""
    gow, g, params = _flat(N, 2)
    g.update_velocity()
    d16, n16 = g.maps_to_host(0, 2)
    maps = (d16, n16, g.velocity_to_host(0, 2))
    assert not d16.astype(np.float32).any()
    yield g, np.ascontiguousarray(gow.WaveGenerator.map_scales(params), np.float32), maps
    g.free()


def _forces_and_simulate(flat, meshes, v, t, fb, s, what):
    """hull_forces on the states' poses and simulate_hull_bodies at S = 1 and 4, each byte-identical to the specification."""
    g, sc, (d16, n16, vel) = flat
    g.set_hull_meshes(meshes, v, t)
    table, bv = oh.pose(fb, s)
    got = g.hull_forces(table, bv, sc, RHO, TOL, 8, return_samples=True)
    with np.errstate(all="ignore"):
        want = oh.hull_forces(d16, n16, vel, table, bv, meshes, v, t, sc, RHO, TOL, 8, True)
    _assert_same(got, want, what + ": hull_forces")
    for S in (1, 4):
        got_s = g.simulate_hull_bodies(fb, s, sc, DT, S, RHO, TOL, 8, return_records=True, return_transforms=True)
        with np.errstate(all="ignore"):
            want_s = oh.simulate(d16, n16, vel, fb, s, meshes, v, t, sc, RHO, DT, S, TOL, 8)
        _assert_same(got_s, want_s, f"{what}: simulate_hull_bodies S = {S}")
    return got


def _floating(meshes, mesh_of, rng=None):
    fb = np.zeros(len(mesh_of), oh.FLOATING)
    fb["mesh"] = mesh_of
    fb["mass"] = 500.0 if rng is None else rng.uniform(100.0, 2000.0, len(mesh_of))
    fb["inertia"] = 200.0 if rng is None else rng.uniform(50.0, 900.0, (len(mesh_of), 3))
    return fb


@pytest.mark.gpu
def test_clip_cases_at_zero_and_subnormal_depths(flat):
    """Every clip case, rotation and winding, with corners at depth exactly 0, +-2^-149, +-1e-40 and +-1e-30: the records
    byte-identical to the specification (the device keeps subnormals, as numpy does), and the pressure force of the exact-zero
    triangles equal to its float64 hand integral."""
    meshes, v, t, heights = _clip_meshes()
    rng = np.random.default_rng(5)
    s = _identity(len(meshes))
    s["linear_velocity"] = rng.normal(size=(len(meshes), 3))
    fb = _floating(meshes, np.arange(len(meshes)))
    hyd, drg, _ = _forces_and_simulate(flat, meshes, v, t, fb, s, "clip cases")
    wet = (heights < 0).sum(1)
    assert {0, 1, 2, 3} <= set(wet.tolist())
    exact = np.all((heights == 0) | (np.abs(heights) >= 0.5), 1)
    assert exact.sum() >= 40
    for m in np.nonzero(exact)[0]:
        p = v[3 * m:3 * m + 3][t[m]]
        want = _hand_force(p)
        np.testing.assert_allclose(hyd["force"][m], want, rtol=2e-6, atol=1e-6 * RHO_G, err_msg=f"mesh {m} heights {heights[m]}")
    assert not hyd["force"][wet == 0].any() and (hyd["force"][wet == 3] != 0).any(axis=1).all()
    # a subnormal wet corner of an otherwise dry triangle is still a (vanishing) wet piece
    sub = (wet == 1) & np.any((heights < 0) & (heights > -1e-37), 1)
    assert sub.any()


@pytest.mark.gpu
def test_degenerate_meshes(flat):
    """A mesh with vertices and no triangles, zero-area triangles with a repeated index, and a mesh whose triangles use only
    some of its vertices (the unused ones still enter max_residual and unconverged), beside an ordinary box."""
    from test_oracle_hull import box
    bv, bt, _ = box(2.0, 1.0, 3.0)
    parts = [(bv, np.zeros((0, 3), np.int32)),                                     # vertices, no triangles
             (bv, np.array([[0, 0, 1], [2, 3, 3], [4, 5, 4]], np.int32)),          # every triangle repeats an index
             (np.concatenate([bv, bv + (0.0, -5.0, 0.0), [[0.0, 9.0, 0.0]]]).astype(np.float32), bt),     # 9 unused vertices
             (bv, bt)]
    meshes = np.zeros(len(parts), oh.MESH)
    fv = ft = 0
    for k, (pv, pt) in enumerate(parts):
        meshes[k] = (fv, len(pv), ft, len(pt), 0.9, 0.1)
        fv, ft = fv + len(pv), ft + len(pt)
    v, t = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    rng = np.random.default_rng(6)
    mesh_of = np.array([0, 1, 2, 3, 0, 2, 1, 3, 2])
    fb = _floating(meshes, mesh_of, rng)
    s = _identity(len(mesh_of), rng, ty=0.1)
    hyd, drg, smp = _forces_and_simulate(flat, meshes, v, t, fb, s, "degenerate meshes")
    assert not hyd["force"][mesh_of <= 1].any() and not drg["wetted_drag_area"][mesh_of <= 1].any()
    assert (hyd["submerged_volume"][mesh_of >= 2] > 0).all()
    assert len(smp) == int(meshes["num_vertices"][mesh_of].sum())


def _ring(n, rng):
    """n vertices on a wavy ring and the n triangles (i, i+1, i+2): a mesh of n triangles on n vertices."""
    th = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = rng.uniform(1.0, 3.0, n)
    v = np.stack([r * np.cos(th), rng.uniform(-1.0, 1.0, n), r * np.sin(th)], 1).astype(np.float32)
    i = np.arange(n)
    return v, np.stack([i, (i + 1) % n, (i + 2) % n], 1).astype(np.int32)


def _lane_meshes(rng):
    """Meshes of 31, 32, 33, 63, 64 and 65 triangles and vertices, then an empty mesh (index 6)."""
    parts = [_ring(n, rng) for n in (31, 32, 33, 63, 64, 65)] + [(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))]
    meshes = np.zeros(len(parts), oh.MESH)
    fv = ft = 0
    for k, (pv, pt) in enumerate(parts):
        meshes[k] = (fv, len(pv), ft, len(pt), rng.uniform(0.2, 1.5), rng.uniform(0.0, 0.2))
        fv, ft = fv + len(pv), ft + len(pt)
    return meshes, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def _random_poses(rng, B):
    s = _identity(B, rng)
    q = rng.normal(size=(B, 4))
    s["orientation"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    s["position"][:, 1] = rng.uniform(-0.8, 0.8, B)
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 7, 8, 9, 17])
def test_lane_and_block_edges(flat, B):
    """Triangle and vertex counts where the 32-lane loops end or wrap, body counts around 8 bodies per block, and empty-mesh
    bodies first, between others and last (repeated offsets for the transform's binary search)."""
    rng = np.random.default_rng(B)
    meshes, v, t = _lane_meshes(rng)
    mesh_of = np.arange(B) % 6
    if B > 1:
        mesh_of[[0, B // 2, B - 1]] = 6
        if B >= 8:
            mesh_of[B // 2 + 1] = 6                             # two empty bodies in a row
    fb = _floating(meshes, mesh_of, rng)
    s = _random_poses(rng, B)
    hyd, drg, _ = _forces_and_simulate(flat, meshes, v, t, fb, s, f"B = {B}")
    empty = mesh_of == 6
    assert not hyd[empty].tobytes().strip(b"\0") and not drg[empty].tobytes().strip(b"\0")
    assert (hyd["force"][~empty] != 0).any()


@pytest.mark.gpu
def test_depths_near_the_binary32_limit(flat):
    """One body at t.y = -3e38 and one at +3e38 among ordinary ones: their moment and force sums overflow to +-inf or NaN as
    the specification's do, and no other body's bytes change."""
    g, sc, (d16, n16, vel) = flat
    rng = np.random.default_rng(9)
    meshes, v, t = _lane_meshes(rng)
    B = 12
    mesh_of = np.arange(B) % 7
    fb = _floating(meshes, mesh_of, rng)
    s = _random_poses(rng, B)
    g.set_hull_meshes(meshes, v, t)
    table, bv = oh.pose(fb, s)
    base = g.hull_forces(table, bv, sc, RHO, TOL, 8, return_samples=True)
    far = table.copy()
    far["transform"][3, 7], far["transform"][8, 7] = -3e38, 3e38
    got = g.hull_forces(far, bv, sc, RHO, TOL, 8, return_samples=True)
    with np.errstate(all="ignore"):
        want = oh.hull_forces(d16, n16, vel, far, bv, meshes, v, t, sc, RHO, TOL, 8, True)
    _assert_same(got, want, "far bodies")
    assert not np.isfinite(got[0]["torque"][3]).all() or not np.isfinite(got[0]["force"][3]).all()
    assert not got[0]["force"][8].any()                         # 3e38 above the water: every corner dry
    keep = np.setdiff1d(np.arange(B), [3, 8])
    for x, y in zip(got[:2], base[:2]):
        assert x[keep].tobytes() == y[keep].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [1e-6, 1.0 / 60.0, 10.0])
def test_integrator_over_its_accepted_range(flat, dt):
    """64 sub-steps, dt from 1e-6 to 10 s, masses and inertias from 1e-3 to 1e9, and non-unit input quaternions (used as
    given for the first sub-step): states, records and transforms byte-identical to the specification."""
    g, sc, (d16, n16, vel) = flat
    rng = np.random.default_rng(int(dt * 1e6) % 1000)
    meshes, v, t = _lane_meshes(rng)
    B = 10
    fb = _floating(meshes, np.arange(B) % 7, rng)
    fb["mass"] = [1e-3, 1e9, 1.0, 1e3, 1e6, 1e-3, 1e9, 50.0, 1e-2, 5e8]
    fb["inertia"] = np.array([[1e-3, 1e9, 1.0], [1e9, 1e9, 1e9], [1e-3, 1e-3, 1e-3], [1.0, 1e3, 1e6], [5.0, 5.0, 5.0],
                              [1e9, 1e-3, 1e2], [1e-3, 1.0, 1e9], [3e2, 3e2, 3e2], [1e6, 1e-3, 1.0], [1e8, 1e8, 1e-3]])
    s = _random_poses(rng, B)
    s["orientation"][::2] *= rng.uniform(0.5, 2.0, (B // 2, 1)).astype(np.float32)     # non-unit quaternions
    assert np.abs(np.linalg.norm(s["orientation"].astype(np.float64), axis=1) - 1).max() > 0.1
    g.set_hull_meshes(meshes, v, t)
    got = g.simulate_hull_bodies(fb, s, sc, dt, 64, RHO, TOL, 8, return_records=True, return_transforms=True)
    with np.errstate(all="ignore"):
        want = oh.simulate(d16, n16, vel, fb, s, meshes, v, t, sc, RHO, dt, 64, TOL, 8)
    _assert_same(got, want, f"dt = {dt}")
