"""The agent key table (csrc/agr_agents.hpp, the code the engine ships, compiled into tests/agent_table_harness.cpp) under agent
churn, on the CPU: random insert / delete / lookup sequences against a Python dict.  Deletion shifts later entries of the probe
cluster back instead of leaving tombstones, so every id stays reachable, the table never fills with dead entries, and a lookup of
a deleted id misses."""
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("agents") / "agent_table_harness")
    res = subprocess.run(["g++", "-O2", "-std=c++17", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "agent_table_harness.cpp")],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr

    def run(cmds):
        out = subprocess.run([exe], input="\n".join(cmds) + "\n", capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        return out.stdout.split("\n")[:-1]
    return run


def churn(run, entries, max_agents, steps, seed):
    """max_agents slots on a table of `entries` (the engine's next_pow2(2 max_agents)); every step deletes a live id or inserts a
    new one onto a free slot, and every id ever used is looked up after it.  Returns the per-step answers for the caller's checks."""
    rng = random.Random(seed)
    live = {}                                       # id -> slot
    free = list(range(max_agents))
    gone = []
    cmds, kinds = [f"n {entries}"], ["n"]
    stats = {"wrapped": 0, "mid": 0, "full": 0}
    for step in range(steps):
        if free and (step < max_agents or not live or rng.random() < 0.55):     # fill up first, then churn
            name = f"agent-{rng.getrandbits(60)}"
            slot = free.pop(rng.randrange(len(free)))
            live[name] = slot
            cmds.append(f"i {name} {slot}"); kinds.append(("i", name))
        else:
            name = rng.choice(sorted(live))
            free.append(live.pop(name)); gone.append(name)
            cmds.append(f"d {name}"); kinds.append(("d", name))
        for name, slot in live.items():
            cmds.append(f"f {name}"); kinds.append(("f", name, slot))
        for name in gone[-8:]:
            if name not in live:
                cmds.append(f"f {name}"); kinds.append(("f", name, None))
        cmds.append("v"); kinds.append(("v", len(live)))
    out = run(cmds)
    assert len(out) == len(kinds)
    for k, o in zip(kinds, out):
        if k == "n":
            assert o == "ok"
        elif k[0] == "i":
            assert 0 <= int(o) < entries
        elif k[0] == "d":
            idx, count = map(int, o.split())
            assert 1 <= count < entries
            stats["mid"] += count > 1                     # the deleted entry had live entries after it in its cluster
        elif k[0] == "f":
            assert o == ("none" if k[2] is None else str(k[2])), k
        else:
            word, n, wrapped = o.split()
            assert word == "ok" and int(n) == k[1], o
            stats["wrapped"] += int(wrapped)
            stats["full"] += int(n) == max_agents
    return stats


@pytest.mark.parametrize("max_agents", [1, 2, 5, 8, 64])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_churn_matches_a_dict(harness, max_agents, seed):
    entries = 1 << max(1, (2 * max_agents - 1).bit_length())
    stats = churn(harness, entries, max_agents, 400, seed * 1000 + max_agents)
    assert stats["full"] > 0                              # the table was at max_agents live keys
    if max_agents >= 5:
        assert stats["wrapped"] > 0 and stats["mid"] > 0  # clusters across the end of the table; deletes inside a cluster


def test_deleting_inside_a_cluster_that_wraps(harness):
    """Ids whose homes are the last entries of a small table: their cluster runs over the end, and deleting each position of it
    in turn keeps the others reachable."""
    entries = 16
    homes = {}
    run = harness
    # find ids by home: the harness places an id alone in an empty table at its home
    for n in range(4000):
        name = f"agent-{n}"
        idx = int(run([f"n {entries}", f"i {name} 0"])[1])
        homes.setdefault(idx, []).append(name)
        if all(len(homes.get(h, [])) >= 2 for h in (13, 14, 15)):
            break
    ids = homes[14][:2] + homes[15][:2] + homes[13][:1]          # cluster 13.. wraps to 0, 1
    for victim in range(len(ids)):
        cmds = [f"n {entries}"] + [f"i {name} {s}" for s, name in enumerate(ids)] + ["v", f"d {ids[victim]}", "v"]
        cmds += [f"f {name}" for name in ids]
        out = run(cmds)
        placed = [int(x) for x in out[1:1 + len(ids)]]
        assert 0 in placed or 1 in placed                         # the cluster wrapped
        assert out[1 + len(ids)].split()[0] == "ok" and out[1 + len(ids)].split()[2] == "1"
        assert out[3 + len(ids)].startswith("ok ")
        assert out[4 + len(ids):] == ["none" if s == victim else str(s) for s in range(len(ids))]
