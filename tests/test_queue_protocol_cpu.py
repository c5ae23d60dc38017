"""The persistent kernel's dependency protocol, run on the CPU against random team schedules (no GPU).

The kernel's teams draw work items from a queue two items ahead of the one they run and synchronise through completion
counters only (DESIGN.md section 4): a column-pass (B) item waits for the row pass (A items) of its cascade; in a fused launch
(ocean_update_frames) the frames alternate between the two halves of the row-pass scratch, a row pass waits for the column pass
two frames back (the last reader of its half) and a column pass additionally for the previous frame's column pass (foam plane).

This test takes the REAL hand-out order (ocean_debug_work_queue) and the REAL wait targets (ocean_debug_frame_protocol -- the
arithmetic ocean_update_frames uses, including the counters' wrap-around) and simulates teams that start, run for a random time
and finish items in a random interleaving.  At every start it checks the ground truth the waits are there to guarantee:
  * a B item starts only when every A item of its (frame, cascade) has finished, and every B item of the previous frame of that
    cascade (it reads that frame's foam and overwrites its maps);
  * an A item starts only when every B item that reads the scratch half it overwrites has finished;
and at the end that every item ran exactly once, nobody waited forever (a schedule in which no team can move is a dead-lock) and
the counters hold what the host mirror says they hold.  The first fused-frame version with ONE row-pass counter per cascade fails
this test in a few hundred steps (a column pass is let through by the next frame's row-pass items); it passed the 1000-frame GPU
oracle test by timing.
"""
import ctypes as C
import random

import numpy as np
import pytest

from godotoceanwaves_b200 import native

M32 = 0xFFFFFFFF


def _reached(seen, target):           # counter_reached() of the kernel: wrap-safe "seen >= target"
    d = (seen - target) & M32
    return d < 0x80000000


def _queue(lib, map_size, count, group, lag, frames):
    total = lib.ocean_debug_work_queue(map_size, count, group, lag, frames, None, 0)
    assert total > 0
    items = (C.c_int32 * total)()
    assert lib.ocean_debug_work_queue(map_size, count, group, lag, frames, items, total) == total
    codes = np.frombuffer(items, dtype=np.int32).astype(np.int64) & M32
    return [(int(c >> 31) & 1, int(c >> 16) & 0x7FFF, int(c) & 0xFFFF) for c in codes]      # (is_b, slot, block)


class Sim:
    """Teams with two items of look-ahead over one launch.  records[slot] = dict(cascade, frame, done_slot, done_target,
    wait_target (A, multi-frame only), col_wait_target (B, multi-frame only))."""

    def __init__(self, items, records, counters, num_cascades, teams, rng, multi_frame, truth):
        self.items, self.rec, self.cnt, self.C = items, records, counters, num_cascades
        self.rng, self.multi, self.truth = rng, multi_frame, truth
        self.next_pos = 0
        self.teams = [dict(held=[self._draw(), self._draw(), self._draw()], state="idle", left=0) for _ in range(teams)]
        self.ran = set()

    def _draw(self):
        p = self.next_pos
        self.next_pos += 1
        return p

    def _can_start(self, it):
        is_b, slot, _ = it
        r = self.rec[slot]
        c = r["cascade"]
        if is_b:
            if self.multi and not _reached(self.cnt[self.C + c], r["col_wait_target"]):
                return False
            return _reached(self.cnt[r["done_slot"]], r["done_target"])
        return (not self.multi) or _reached(self.cnt[self.C + c], r["wait_target"])

    def step(self):
        """One scheduling decision; returns False when every team is finished, raises on a dead-lock."""
        movable, busy = [], False
        for t in self.teams:
            pos = t["held"][0]
            if pos >= len(self.items):
                continue
            busy = True
            if t["state"] == "running" or self._can_start(self.items[pos]):
                movable.append(t)
        if not busy:
            return False
        assert movable, "dead-lock: every team waits for a counter nobody is going to bump"
        t = self.rng.choice(movable)
        it = self.items[t["held"][0]]
        if t["state"] == "idle":
            self.truth.on_start(it, self.rec[it[1]])
            t["state"], t["left"] = "running", self.rng.randint(0, 3)
        elif t["left"] > 0:
            t["left"] -= 1
        else:                                           # finish: release the counter, move on, draw one more position
            is_b, slot, _ = it
            r = self.rec[slot]
            key = r["cascade"] + self.C if is_b else r["done_slot"]
            self.cnt[key] = (self.cnt[key] + 1) & M32
            self.truth.on_finish(it, r)
            assert it not in self.ran
            self.ran.add(it)
            t["held"].pop(0)
            t["held"].append(self._draw())
            t["state"] = "idle"
        return True

    def run(self):
        steps = 0
        while self.step():
            steps += 1
            assert steps < 5_000_000
        assert len(self.ran) == len(self.items)


class Truth:
    """What has really finished, per (kind, frame, cascade) -- independent of the counters."""

    def __init__(self, a_per, b_per):
        self.a_per, self.b_per = a_per, b_per
        self.fin = {}           # (kind, frame, cascade) -> finished items
        self.started_a = {}     # (frame, cascade) -> started row-pass items (they overwrite the scratch half)

    def done(self, kind, frame, cascade):
        per = self.b_per if kind else self.a_per
        return self.fin.get((kind, frame, cascade), 0) == per

    def on_start(self, it, r):
        is_b, _, _ = it
        f, c = r["frame"], r["cascade"]
        if is_b:
            assert self.done(0, f, c), f"column pass of frame {f}, cascade {c} starts on an unfinished row pass"
            if f - 1 >= r["first_frame"]:           # (earlier launches are complete when this one starts)
                assert self.done(1, f - 1, c), f"column pass of frame {f} starts before the foam of frame {f - 1} is complete"
            # nobody may already be overwriting the half this item reads: the row pass two frames on
            assert self.started_a.get((f + 2, c), 0) == 0
        else:
            if f - 2 >= r["first_frame"]:
                assert self.done(1, f - 2, c), f"row pass of frame {f}, cascade {c} overwrites a scratch half that is still being read"
            self.started_a[(f, c)] = self.started_a.get((f, c), 0) + 1

    def on_finish(self, it, r):
        k = (it[0], r["frame"], r["cascade"])
        self.fin[k] = self.fin.get(k, 0) + 1


def default_queue(map_size):
    """(group, lag) of persistent_group / persistent_lag without overrides: two thirds of an L2-sized chunk of the two-kernel
    pipeline per group (chunk_cascades: 24 MiB of scratch at 32 B per texel), lag 2 at 1024^2."""
    chunk = max(1, (24 << 20) // (map_size * map_size * 32))
    return max(1, chunk * 2 // 3), (2 if map_size >= 1024 else 1)


def batch_queue_shapes():
    """The queue shapes tests/test_gpu_batch_shapes.py forces on the GPU through OCEAN_QUEUE_GROUP / OCEAN_QUEUE_LAG, as
    (map_size, count, name, group, lag) with None for "no override": per size the default, the most waits (group 1, lag 1),
    a group that does not divide the count (a short last group), one group, a lag beyond the number of groups (every row
    pass before any column pass) and lag 3.  At 256^2 x 24 the default makes 3 groups, at 128^2 x 70 groups of 32, 32
    and 6, at 512^2 x 7 groups of 2, 2, 2 and 1, and 1024^2 x 8 is cfg4-strong's shape on one GPU (group 1, lag 2)."""
    out = []
    for N, C in ((256, 24), (128, 70), (512, 7), (1024, 8)):
        short = next(g for g in range(3, C) if C % g)
        out += [(N, C, "default", None, None), (N, C, "group1_lag1", 1, 1), (N, C, "short_last_group", short, None),
                (N, C, "single_group", C + 1, None), (N, C, "every_row_pass_first", None, 64), (N, C, "lag3", None, 3)]
    return out


def _resolved(shape):
    N, C, _, group, lag = shape
    dg, dl = default_queue(N)
    return N, C, group or dg, lag or dl


@pytest.mark.parametrize("map_size,count,group,lag,teams,seed", [
    (256, 9, 2, 1, 7, 1), (256, 9, 2, 3, 5, 2), (128, 6, 1, 1, 3, 3), (128, 7, 3, 4, 11, 4), (256, 20, 16, 1, 23, 5), (512, 5, 0, 0, 6, 6),
    (256, 128, 8, 1, 33, 100)]                                  # the bench workload: 16 groups of 8 cascades, lag 1
    + [(*_resolved(s), 4 + (13 * k) % 41, 101 + k) for k, s in enumerate(batch_queue_shapes())])
def test_single_update_protocol_under_random_schedules(map_size, count, group, lag, teams, seed):
    lib = native.load_library()
    items = _queue(lib, map_size, count, group, lag, 0)
    a_per = sum(1 for b, s, _ in items if not b and s == 0)
    b_per = sum(1 for b, s, _ in items if b and s == 0)
    rng = random.Random(seed)
    counters = [(M32 - rng.randint(0, 3 * a_per)) & M32 for _ in range(3 * count)]          # close to the wrap-around
    records = {c: dict(cascade=c, frame=0, first_frame=0, done_slot=c,
                       done_target=(counters[c] + a_per) & M32) for c in range(count)}       # run_cascades: done_count[i] + per_update
    start = list(counters)
    sim = Sim(items, records, counters, count, teams, rng, multi_frame=False, truth=Truth(a_per, b_per))
    sim.run()
    for c in range(count):
        assert counters[c] == (start[c] + a_per) & M32


@pytest.mark.parametrize("map_size,num_cascades,count,launches,teams,seed", [
    (256, 4, 4, [3, 2], 7, 1), (256, 4, 4, [5], 13, 2), (512, 4, 4, [4, 4, 1], 9, 3), (128, 3, 2, [1, 2, 6], 4, 4), (1024, 8, 8, [2, 3], 10, 5),
    # full dispatch tables of 256 records: 4 frames of 64 cascades and 2 frames of the bench workload's 128 per launch
    (256, 64, 64, [4, 4, 1], 29, 6), (256, 128, 128, [2, 2], 37, 7)])
def test_fused_frames_protocol_under_random_schedules(map_size, num_cascades, count, launches, teams, seed):
    lib = native.load_library()
    rng = random.Random(seed)
    CN = num_cascades
    mirror = (C.c_uint32 * (3 * CN))(*[(M32 - rng.randint(0, 200)) & M32 for _ in range(3 * CN)])    # host mirror, close to the wrap
    counters = list(mirror)                                                                           # the device's counters
    first_frame = 1                                   # frame 0 of a call is an ordinary update in half 0 (ocean_update_all)
    truth = None
    for F in launches:
        items = _queue(lib, map_size, count, 0, 0, F)
        a_per = sum(1 for b, s, _ in items if not b and s == 0)
        b_per = sum(1 for b, s, _ in items if b and s == 0)
        rec = (C.c_int32 * (F * count * 6))()
        assert lib.ocean_debug_frame_protocol(map_size, CN, count, first_frame, F, mirror, rec) == 0
        r = np.frombuffer(rec, dtype=np.int32).reshape(F * count, 6).astype(np.int64) & M32
        records = {}
        for slot in range(F * count):
            f, c = divmod(slot, count)
            assert int(r[slot, 0]) == c
            half = (first_frame + f) & 1
            assert int(r[slot, 1]) == (2 * CN + c if half else c) and int(r[slot, 5]) == 2 * (half * CN + c)
            records[slot] = dict(cascade=c, frame=first_frame + f, first_frame=first_frame,
                                 done_slot=int(r[slot, 1]), done_target=int(r[slot, 2]), wait_target=int(r[slot, 3]),
                                 col_wait_target=int(r[slot, 4]))
        truth = Truth(a_per, b_per)                   # every frame of earlier launches is complete when a launch starts
        Sim(items, records, counters, CN, teams, rng, multi_frame=True, truth=truth).run()
        assert counters == list(mirror), "the host mirror of the completion counters disagrees with what the items bumped"
        first_frame += F


def test_one_counter_for_both_halves_would_race():
    """The negative control: with a single row-pass counter per cascade (the first fused-frame version) the same simulation finds
    a column pass that starts on an unfinished row pass -- i.e. the check above can fail."""
    lib = native.load_library()
    map_size, CN, count, F = 256, 2, 2, 6
    items = _queue(lib, map_size, count, 0, 0, F)
    a_per = sum(1 for b, s, _ in items if not b and s == 0)
    b_per = sum(1 for b, s, _ in items if b and s == 0)
    found = False
    for seed in range(40):
        rng = random.Random(seed)
        counters = [0] * (3 * CN)
        records = {}
        for slot in range(F * count):
            f, c = divmod(slot, count)
            records[slot] = dict(cascade=c, frame=1 + f, first_frame=1, done_slot=c,
                                 done_target=(f + 1) * a_per, wait_target=max(0, f - 1) * b_per, col_wait_target=f * b_per)
        try:
            Sim(items, records, counters, CN, 37, rng, multi_frame=True, truth=Truth(a_per, b_per)).run()
        except AssertionError as e:
            if "unfinished row pass" in str(e):
                found = True
                break
    assert found
