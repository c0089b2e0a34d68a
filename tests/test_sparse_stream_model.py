"""CPU: the numpy model of SparseTsdfVolume's streaming policy (tests/sparse_stream_model.py) on a case worked out by hand,
its invariants on the ring walks, and what the scenes the GPU tests stream exercise: an edit to a scene or a budget that
loses one of these cases fails here."""
import numpy as np
import pytest

import sequence_oracle as so
import sparse_stream_model as sm
import sparse_stream_oracle as ss
import sparse_tsdf_oracle as sp

f32 = np.float32


def patch_view(y):
    """One 8x8 frame of a camera at (0, y, 0.5) looking along +x at a wall 3 m away: a few blocks at voxel 0.1, far enough
    in front that no widened block straddles the camera plane."""
    R, t = so.look_at(np.array([0.0, y, 0.5]), np.array([1.0, y, 0.5]))
    K = np.array([[100.0, 0, 4.0], [0, 100.0, 4.0], [0, 0, 1]], f32)
    return np.full((1, 8, 8), 3.0, f32), K[None], np.asarray(R, f32)[None], np.asarray(t, f32)[None]


def test_three_regions_and_a_return():
    """Budget 2; calls 1-3 allocate disjoint regions A, B, C that no other call reaches; call 4 integrates call 1's frame
    again.  Worked out from the policy, with A, B, C in key order and a, b, c their sizes:
      call 1: A[:a-2] leave (stamp 1, ties by key) for slots 0..a-3; A[a-2:] stay.
      call 2: A[a-2:] (stamp 1) leave before B[:b-2] (stamp 2); B[b-2:] stay.  Host: A, B[:b-2].
      call 3: likewise.  Host: A, B, C[:c-2].
      call 4: A comes back from slots 0..a-1 and is appended; C[c-2:] (stamp 3, not reached) leave first, into the
              lowest free slots 0 and 1, then A[:a-2] (stamp 4) into slots 2..a-1; A[a-2:] stay."""
    vs, origin = 0.1, (0.013, -0.021, 0.007)
    trunc = f32(3 * f32(vs))
    views = [patch_view(y) for y in (0.0, 12.0, 20.0)]
    A, B, C = regions = [sorted(sp.allocate(*v, origin, vs, trunc)[0], key=sm.key_order) for v in views]
    a, b, c = (len(r) for r in regions)
    assert min(a, b, c) >= 3 and len(set(A) | set(B) | set(C)) == a + b + c
    for i, (d, K, R, t) in enumerate(views):   # each camera reaches its own region and no other
        for j, r in enumerate(regions):
            hit = ss.reach(sm.as_blocks(r), origin, vs, trunc, ss.depth_tiles(d), K, R, t, 8, 8)[0]
            assert hit.all() if i == j else not hit.any(), (i, j)
    model = sm.StreamModel(2, origin, vs, trunc, color=False)

    def check(device, host, bin_, bout, peak):
        st = model.state()
        assert [tuple(x) for x in st["blocks"].tolist()] == device
        assert [tuple(x) for x in st["host"].tolist()] == host
        assert (st["last_blocks_in"], st["last_blocks_out"], st["peak_device_blocks"]) == (bin_, bout, peak)

    model.integrate(*views[0])
    check(A[a - 2:], A[:a - 2], 0, a - 2, a)
    assert model.slots == A[:a - 2]
    model.integrate(*views[1])
    check(B[b - 2:], A + B[:b - 2], 0, b, max(a, b + 2))
    model.integrate(*views[2])
    check(C[c - 2:], A + B + C[:c - 2], 0, c, max(a, b + 2, c + 2))
    assert model.host_capacity == sm.doubling(1, a + b + c - 2)
    assert model.host_nbytes == 4096 * model.host_capacity
    model.integrate(*views[0])
    check(A[a - 2:], C[c - 2:] + A[:a - 2] + B + C[:c - 2], a, a, max(a + 2, b + 2, c + 2))
    assert model.slots == C[c - 2:] + A[:a - 2] + B + C[:c - 2]   # no slot left free
    assert model.stamp == {x: 4 for x in A[a - 2:]}
    rec = model.log[-1]
    assert rec["evicted_unreached_kept_reached"] and rec["reused_freed"] and rec["stamps"] == {3, 4}


def test_free_slots_at_the_end_are_trimmed_and_the_lowest_reused():
    """Budget 2 with four regions: bringing back the region in the last slots shortens the store, and bringing back one
    in the middle leaves a hole that the next eviction fills lowest first."""
    vs, origin = 0.1, (0.013, -0.021, 0.007)
    trunc = f32(3 * f32(vs))
    views = [patch_view(y) for y in (0.0, 12.0, 20.0, 32.0)]
    model = sm.StreamModel(2, origin, vs, trunc, color=True)
    for v in views:
        model.integrate(*v)
    used = len(model.slots)
    D = sorted(sp.allocate(*views[3], origin, vs, trunc)[0], key=sm.key_order)
    assert model.slots[-(len(D) - 2):] == D[:len(D) - 2]
    model.raycast(*views[3][1:], 8, 8, far=4.0)   # D[:-2] comes back from the end of the store, 2 other blocks leave
    assert model.last_blocks_in == len(D) - 2 and model.last_blocks_out == len(D) - 2
    assert len(model.slots) == used and None not in model.slots
    assert model.host_nbytes == 10240 * model.host_capacity
    B = sorted(sp.allocate(*views[1], origin, vs, trunc)[0], key=sm.key_order)
    lo = model.slots.index(B[0])
    model.raycast(*views[1][1:], 8, 8, far=4.0)   # B comes back from the middle: B[:2] stay, the rest of B and 2 leave
    assert model.last_blocks_in == len(B)
    assert all(model.slots[s] is not None for s in range(len(model.slots)))
    assert model.slots[lo:lo + 2] == model.log[-1]["evicted"][:2]


@pytest.fixture(scope="module", params=["A", "B"])
def scene(request):
    frames, per_call = sm.scene(request.param)
    return request.param, frames, per_call, sm.budgets(frames, per_call)


def test_walk_invariants(scene):
    """After every call the device holds at most the budget, device and host together hold every block allocated so far
    once, and a budget of every block moves nothing."""
    name, frames, per_call, budgets = scene
    allocated = set()
    calls = sm.chunks(frames, per_call)
    for kind, budget in budgets.items():
        states, model = sm.walk(frames, per_call, budget)
        allocated = set()
        for (d, K, R, t, _), st in zip(calls, states):
            allocated |= sp.allocate(d, K, R, t, sm.ORIGIN, sm.VS, sm.TRUNC)[0]
            dev, host = [set(map(tuple, st[k].tolist())) for k in ("blocks", "host")]
            assert st["blocks"].shape[0] <= budget, kind
            assert len(dev) + len(host) == st["blocks"].shape[0] + st["host"].shape[0] and not dev & host
            assert dev | host == allocated, kind
            assert st["table"] >= 2 * len(allocated) and st["capacity"] >= st["blocks"].shape[0]
        assert model.peak_device_blocks > budget, kind
    states, model = sm.walk(frames, per_call, len(allocated))
    assert all(st["last_blocks_in"] == st["last_blocks_out"] == st["host"].shape[0] == st["host_nbytes"] == 0 for st in states)
    assert model.peak_device_blocks == len(allocated)


def test_gpu_scenes_reach_the_policy_cases():
    """The walks and the interleaved calls that tests/test_gpu_sparse_stream_policy.py streams exercise every case of the
    policy that a wrong implementation could get wrong without changing the fused voxels."""
    logs, one = [], {}
    for name in ("A", "B"):
        frames, per_call = sm.scene(name)
        budgets = sm.budgets(frames, per_call)
        for kind, budget in budgets.items():
            _, model = sm.walk(frames, per_call, budget)
            logs += model.log
            one[name] = model if kind == "one" else one.get(name)
        if name == "A":
            _, model = sm.run_interleaved(frames, per_call, budgets["tenth"])
            inter = model.log
            logs += inter
    evictions = [r for r in logs if r["evicted"]]
    assert any(len(r["stamps"]) >= 3 for r in evictions)                     # least recently reached among 3+ stamps
    assert any(r.get("evicted_unreached_kept_reached") for r in evictions)    # not key order over the whole device
    assert any(r["slot_order_differs"] for r in logs if r["kind"] == "integrate")   # key order is not slot order
    assert any(r["slot_order_differs"] for r in inter if r["kind"] == "raycast")
    assert any(r["kind"] == "raycast" and r["evicted"] and r["freed"] for r in inter)   # a ray cast alone brings blocks back
    assert any(r["reused_freed"] for r in logs)                               # slots freed by a call reused in that call
    assert any(r["table_grew"] and r["host_at_start"] for r in logs)          # the table doubles with blocks on the host
    caps = [r["host_capacity"] for r in one["A"].log if "host_capacity" in r]
    assert len(set(caps)) >= 3 and caps == sorted(caps)                       # the budget-1 store doubles several times
    assert len(set(r["host_capacity"] for r in one["B"].log if "host_capacity" in r)) >= 3
