"""The persistent kernel's self-resetting work counter, run on the CPU against random team schedules (no GPU).

Thread 0 of a team takes two tickets (atomicAdd on the counter) before its first item and one more at the start of every item
it runs; it stops when the item it holds is past the end of the queue.  So a launch takes exactly total + 2 * grid tickets, and
take_ticket() (ocean_kernels.cu) lets the holder of the last one put the counter back to 0: the next update's launch finds it
at 0 without a memset between the two launches.  This test restates that discipline over consecutive launches of different
sizes (grids smaller and larger than the queue) and random interleavings of the teams' tickets, and checks:
  * every queue position of every launch is run exactly once;
  * the reset is the last access to the counter in its launch, and every launch starts at 0;
  * every team has taken a ticket past the end before it leaves (it has let a dependent launch begin).
A negative control resets on the first ticket past the end, which a still-running team's next ticket then re-issues.
"""
import random

import pytest

RESIDENT = 396          # 132 SMs x 3 teams at 256^2


def run_launch(counter, total, grid, rng, reset_at):
    """One launch against `counter` (a one-element list); returns the multiset of positions that ran."""
    ran, teams = [], []

    def ticket(team):
        t = counter[0]
        counter[0] += 1
        if t >= total:
            team["triggered"] = True
            if t == reset_at(total, grid):
                counter[0] = 0
                team["reset"] = True
        return t

    for _ in range(grid):
        teams.append(dict(held=[], triggered=False, reset=False, phase="prologue"))
    live = list(teams)
    resets = 0
    while live:
        team = rng.choice(live)
        if team["phase"] == "prologue":            # two tickets, possibly interleaved with other teams'
            team["held"].append(ticket(team))
            if len(team["held"]) == 2:
                team["phase"] = "loop"
        else:
            cur = team["held"].pop(0)
            if cur >= total:                        # code == -1: the team leaves
                assert team["triggered"], "a team left without having let the dependent launch begin"
                live.remove(team)
                continue
            team["held"].append(ticket(team))       # the ticket of the item after the next
            ran.append(cur)
        resets += team.pop("reset", False)
        team["reset"] = False
    return ran, resets


@pytest.mark.parametrize("seed", range(4))
def test_consecutive_launches_share_one_counter(seed):
    rng = random.Random(seed)
    counter = [0]
    last = lambda total, grid: total + 2 * grid - 1
    for _ in range(20):
        total = rng.choice([12288, 6144, 96, 3, 1, 500, RESIDENT, RESIDENT + 1])
        grid = min(total, RESIDENT)
        assert counter[0] == 0, "a launch started with a non-zero work counter"
        ran, resets = run_launch(counter, total, grid, rng, last)
        assert sorted(ran) == list(range(total)), "queue positions lost or run twice"
        assert resets == 1
        assert counter[0] == 0, "the counter was touched after its reset"


def test_reset_before_the_last_ticket_fails():
    """Negative control: resetting on the first ticket past the end hands some positions out twice."""
    rng = random.Random(1)
    counter = [0]
    early = lambda total, grid: total
    with pytest.raises(AssertionError):
        for _ in range(10):
            ran, _ = run_launch(counter, 6144, RESIDENT, rng, early)
            assert sorted(ran) == list(range(6144)) and counter[0] == 0
