"""Which kernels the batched world launches, on the CPU: a mirror of the dispatch of nb_world_scan and nb_world_step
(csrc/world_api.cu), the table of every kernel instantiation those two entry points name, and MATRIX, the named configurations
that tests/test_gpu_world_variants.py runs against the float64 oracles.  Together the configurations must reach every
instantiation: a new switch in the dispatch adds kernels to the source, this test then fails until the table, the mirror and
MATRIX cover them."""
import itertools
import os
import re

import pytest

from neupan_b200.world import pack_behaviors, pack_map_contact, pack_obstacle_contact
from test_gpu_world_contact import _contact_scenes
from test_gpu_world_mixed import _robot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ("ep", "map", "blocking", "contact", "act", "rvo", "noise")
B2 = (False, True)


def kernel(name, *args):
    """A kernel's name with its template arguments, as the C++ source spells them."""
    return f"{name}<{', '.join('true' if a else 'false' for a in args)}>" if args else name


# every instantiation that nb_world_scan and nb_world_step name, written out (not derived from the mirror below)
INSTANTIATIONS = frozenset(
    [kernel("world_scan_kernel", m, e, n) for m in B2 for e in B2 for n in B2]
    + [kernel("world_step_kernel", m) for m in B2] + [kernel("world_step_ep_kernel", m) for m in B2]
    + [kernel("world_step_block_kernel", e) for e in B2]
    + [kernel("world_step_contact_kernel", m, e) for m in B2 for e in B2]
    + [kernel("world_step_act_kernel", *a) for a in ((False, False, False, False), (True, False, False, False), (False, True, False, False),
                                                      (True, True, False, False), (False, False, False, True), (True, False, False, True),
                                                      (False, True, False, True), (True, True, False, True), (True, False, True, True),
                                                      (True, True, True, True))]
    + [kernel("world_contact_kernel", b, e) for b in B2 for e in B2]
    + [kernel("world_rvo_kernel", e) for e in B2] + [kernel("world_rvo_block_kernel", e) for e in B2])


def accepted(ep, map, blocking, contact, act, rvo, noise):
    """Flags a handle can have: a map that blocks obstacles needs maps (nb_world_set_map_contact refuses a handle without them);
    episodes, obstacle contact, reactive obstacles, actuation and lidar noise combine with anything."""
    return map or not blocking


def dispatch(ep, map, blocking, contact, act, rvo, noise):
    """(step, scan): the kernels one nb_world_step and one nb_world_scan launch, in launch order, for a handle's flags -- the branch
    structure of world_api.cu.  ep: nb_world_set_episodes; map: an environment has a map; blocking: a map blocks obstacles; contact:
    obstacle contact; act: nb_world_set_actuation; rvo: a reactive obstacle; noise: range_std > 0.  Each list's length is the call's
    launch count (nb_launch_count)."""
    scan = [kernel("world_scan_kernel", map, ep, noise)]
    step = []
    if rvo:
        step.append(kernel("world_rvo_block_kernel" if blocking else "world_rvo_kernel", ep))
    if contact:
        step.append(kernel("world_contact_kernel", blocking, ep))
        step.append(kernel("world_step_act_kernel", map, ep, False, False) if act else kernel("world_step_contact_kernel", map, ep))
    elif act:
        step.append(kernel("world_step_act_kernel", True, ep, True, True) if blocking else kernel("world_step_act_kernel", map, ep, False, True))
    elif blocking:
        step.append(kernel("world_step_block_kernel", ep))
    else:
        step.append(kernel("world_step_ep_kernel" if ep else "world_step_kernel", map))
    if ep:
        step.append("world_advance_kernel")
    return step, scan


# ---- the configurations ------------------------------------------------------------------------------------------------------
# scenes: which parts of _contact_scenes (tests/test_gpu_world_contact.py: maps in 7 of 8 environments, blocking in 3 of 4 of those,
# obstacle contact in 7 of 8, circles, polygons and outlines, about half of them reactive) a configuration keeps
SCENES = {
    "free": dict(map=False, blocking=False, contact=False),
    "map": dict(map=True, blocking=False, contact=False),
    "block": dict(map=True, blocking=True, contact=False),
    "contact": dict(map=False, blocking=False, contact=True),
    "contact_map": dict(map=True, blocking=False, contact=True),
    "contact_block": dict(map=True, blocking=True, contact=True),
}
# the plain configurations: scenes, reactive obstacles, nb_world_set_actuation, lidar range noise
PLAIN = {
    "free": ("free", False, False, False),
    "free_rvo_noise": ("free", True, False, True),
    "map_rvo": ("map", True, False, False),
    "block_rvo": ("block", True, False, False),
    "block_noise": ("block", False, False, True),
    "contact_rvo": ("contact", True, False, False),
    "contact_map_noise": ("contact_map", False, False, True),
    "contact_block_rvo_noise": ("contact_block", True, False, True),
    "act": ("free", True, True, False),
    "act_map_noise": ("map", True, True, True),
    "act_block": ("block", True, True, False),
    "act_contact_noise": ("contact", True, True, True),
    "act_contact_map": ("contact_map", False, True, False),
    "act_contact_block_noise": ("contact_block", True, True, True),
}
# every plain configuration also runs as an episode bank ("ep_" + its name)
MATRIX = {**{n: dict(scenes=s, rvo=r, act=a, noise=z, ep=False) for n, (s, r, a, z) in PLAIN.items()},
          **{"ep_" + n: dict(scenes=s, rvo=r, act=a, noise=z, ep=True) for n, (s, r, a, z) in PLAIN.items()}}
# plain runs: a mixed fleet of K = 3; banks: K = 2 diff robots (robot k keeps its type across the bank's scenes)
FLEETS = {False: (("diff", "acker", "omni"), 3), True: (("diff",), 2)}


def variant_scenes(name, B, seed=31):
    """(scenes, robots, K) of MATRIX[name] for B environments: _contact_scenes without the maps, the blocking or the obstacle
    contact the configuration drops, and without the obstacles' behaviours (reactive obstacles then stand still) unless it has
    reactive obstacles.  A bank's scene s with s % 3 == 0 puts every robot's goal at its start (an arrival at step 1)."""
    cfg = MATRIX[name]
    want = SCENES[cfg["scenes"]]
    names, K = FLEETS[cfg["ep"]]
    robots = [_robot(n) for n in names]
    scenes = _contact_scenes(B, K, seed, robots)
    for s, sc in enumerate(scenes):
        if not want["map"]:
            sc.pop("map", None)
        elif not want["blocking"] and "map" in sc:
            sc["map"]["blocks_obstacles"] = False
        if not want["contact"]:
            sc.pop("obstacle_contact", None)
        if not cfg["rvo"]:
            for ob in sc["obstacles"]:
                if ob.pop("behavior", None) is not None:
                    ob["velocity"] = (0.0, 0.0)
        if cfg["ep"] and s % 3 == 0:
            for r in sc["robots"]:
                r["goal"], r["goal_threshold"] = tuple(r["start"][:2]), 1.0
    return scenes, robots, K


def flags_of(name, scenes):
    """The dispatch flags a world gets from MATRIX[name]'s settings and from its scenes, read the way WorldBatch.set_scenes reads
    them."""
    cfg = MATRIX[name]
    has = lambda key: any(key in sc for sc in scenes)
    beh = pack_behaviors(scenes) if any("behavior" in ob for sc in scenes for ob in sc["obstacles"]) else None
    return dict(ep=cfg["ep"], map=has("map"), blocking=has("map") and bool(pack_map_contact(scenes).any()),
                contact=has("obstacle_contact") and bool(pack_obstacle_contact(scenes).any()), act=cfg["act"],
                rvo=beh is not None and bool((beh[:, 0] == 1.0).any()), noise=cfg["noise"])


# B of the GPU tests: plain runs and banks
B_PLAIN, B_BANK = 32, 24


def _source_instantiations():
    """The kernel instantiations named in nb_world_scan and nb_world_step, with the scan's default kNoise = false spelt out."""
    src = open(os.path.join(ROOT, "neupan_b200", "csrc", "world_api.cu")).read()
    body = src[src.index("int nb_world_scan("):src.index("int nb_world_read_state(")]
    found = set()
    for name, args in re.findall(r"nb::(world_\w+_kernel)<([^<>]*)>", body):
        args = [a.strip() for a in args.split(",")]
        if name == "world_scan_kernel" and len(args) == 2:
            args.append("false")
        found.add(f"{name}<{', '.join(args)}>")
    return found


def test_the_table_is_every_instantiation_the_dispatch_names():
    assert len(INSTANTIATIONS) == 36
    src = _source_instantiations()
    assert src == set(INSTANTIATIONS), (sorted(src - INSTANTIATIONS), sorted(INSTANTIATIONS - src))


def test_every_accepted_flag_combination_launches_kernels_of_the_table():
    """Each of the 96 accepted combinations launches kernels of the table only, one scan kernel, and per step its stage kernels plus
    the advance in episode mode; every instantiation is reachable from some combination."""
    reached, combos = set(), 0
    for values in itertools.product(B2, repeat=len(FLAGS)):
        f = dict(zip(FLAGS, values))
        if not accepted(**f):
            continue
        combos += 1
        step, scan = dispatch(**f)
        body = [k for k in step if k != "world_advance_kernel"]
        assert set(body + scan) <= INSTANTIATIONS, (f, set(body + scan) - INSTANTIATIONS)
        assert len(scan) == 1
        assert len(step) == 1 + f["rvo"] + f["contact"] + f["ep"], f
        assert (step[-1] == "world_advance_kernel") == f["ep"], f
        reached |= set(body + scan)
    assert combos == 96
    assert reached == INSTANTIATIONS, sorted(INSTANTIATIONS - reached)


def test_dispatch_examples():
    """A few combinations spelt out by hand."""
    assert dispatch(False, False, False, False, False, False, False) == (["world_step_kernel<false>"], ["world_scan_kernel<false, false, false>"])
    assert dispatch(True, True, True, False, True, True, True) == (
        ["world_rvo_block_kernel<true>", "world_step_act_kernel<true, true, true, true>", "world_advance_kernel"],
        ["world_scan_kernel<true, true, true>"])
    # with obstacle contact the contact kernel moves the obstacles, a blocking map included: the step does not block again
    assert dispatch(False, True, True, True, True, False, False)[0] == ["world_contact_kernel<true, false>",
                                                                       "world_step_act_kernel<true, false, false, false>"]
    assert dispatch(True, True, False, True, False, True, False)[0] == ["world_rvo_kernel<true>", "world_contact_kernel<false, true>",
                                                                        "world_step_contact_kernel<true, true>", "world_advance_kernel"]


@pytest.fixture(scope="module")
def matrix_flags():
    return {n: flags_of(n, variant_scenes(n, B_BANK if cfg["ep"] else B_PLAIN)[0]) for n, cfg in MATRIX.items()}


def test_matrix_scenes_have_the_flags_their_names_promise(matrix_flags):
    for n, f in matrix_flags.items():
        cfg = MATRIX[n]
        assert {k: f[k] for k in ("map", "blocking", "contact")} == SCENES[cfg["scenes"]], n
        assert f["rvo"] == cfg["rvo"], n


def test_matrix_reaches_every_instantiation(matrix_flags):
    reached = {}
    for n, f in matrix_flags.items():
        step, scan = dispatch(**f)
        for k in step + scan:
            reached.setdefault(k, []).append(n)
    missing = sorted(INSTANTIATIONS - set(reached))
    assert not missing, f"no configuration of MATRIX launches {missing}"
