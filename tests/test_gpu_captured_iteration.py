"""``train.CapturedIteration`` and the live line-of-sight constants on the GPU.

1. The live ray-loss entries against the float entries: bit-identical value and gradient over an epsilon sweep from 6.0
   to 2.5 and several decay weights at 2^16 + 17 rays x 64 samples; in a CUDA graph, constants rewritten between
   replays give exactly what eager float calls with those values give.
2. One iteration from a snapshot, for each variant (and ``flow`` with ``EMER_FLOW_BRANCH=fused``): once both of the
   step's keys have been captured, the replayed iteration against the eager restatement of the loop
   (captured_iteration_cases.reference_iteration) from the same parameters, optimizer state, schedulers and CPU / CUDA
   generators.  The pixel pass's logged values are bit-identical.  The lidar pass's values, the parameters and the
   Adam moments agree within 1e-4 relative, or within twice the spread of twelve eager runs from the same snapshot
   where the eager runs themselves spread further (float atomics sum in an order that depends on scheduling, and Adam
   magnifies that on gradients that are cancellation residues; see ``_eager_runs``).  The generator states, learning
   rates and Adam step counters are equal.
3. A 60-iteration trajectory through every branch (line of sight from step 10, decay every 7 steps, an error-map
   refresh at step 20): the expected eager / capture / replay / drop sequence, the exact lr, epsilon and decay weight,
   no host sync and no Python-side library launch in an iteration that only replays, and every drained value within a
   tolerance derived from the spread between two eager trajectories.
4. All graphs share one memory pool; the reserved memory after capture is reported next to the eager peak.
"""
import copy
import math
import warnings

import pytest
import torch

import captured_iteration_cases as cic
from helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ----------------------------------------------------------------------------- 1. live constants
def _float_call(w, t, gt, eps, decay):
    from emernerf_b200 import loss

    w = w.detach().requires_grad_(True)
    v = loss.LineOfSightLoss(coef=0.1)(None, gt, w, t, eps, coef_decay=decay)["line_of_sight_my"]
    v.backward()
    return v.detach(), w.grad


def _live_call(w, t, gt, consts):
    from emernerf_b200 import loss

    w = w.detach().requires_grad_(True)
    v = loss.LineOfSightLoss(coef=0.1)(None, gt, w, t, consts)["line_of_sight_my"]
    v.backward()
    return v.detach(), w.grad


def _rays(n=(1 << 16) + 17, s=64, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    gt = torch.rand(n, device=DEV, generator=g) * 60.0
    gt[::13] = 0.0                                            # rays without a return
    t = torch.sort(torch.rand(n, s, device=DEV, generator=g) * 80.0, dim=-1).values
    w = torch.rand(n, s, device=DEV, generator=g) / s
    return w, t, gt


def test_live_constants_are_bit_identical_to_the_float_entries():
    from emernerf_b200 import loss

    w, t, gt = _rays()
    consts = torch.empty(4, dtype=torch.float32, device=DEV)
    for eps in (6.0, 5.125, 4.3, 3.7, 2.9, 2.5):
        for decay in (1.0, 0.5, 0.25, 0.1 ** 3):
            consts.copy_(torch.tensor(loss.line_of_sight_consts(eps, decay)))
            v_f, g_f = _float_call(w, t, gt, eps, decay)
            v_l, g_l = _live_call(w, t, gt, consts)
            assert torch.equal(v_f, v_l), (eps, decay)
            assert torch.equal(g_f, g_l), (eps, decay)


def test_live_constants_follow_rewrites_between_replays():
    from emernerf_b200 import loss

    w, t, gt = _rays(n=4099, s=64, seed=1)
    w_in = w.clone().requires_grad_(True)
    consts = torch.tensor(loss.line_of_sight_consts(6.0, 1.0), device=DEV)
    fn = loss.LineOfSightLoss(coef=0.1)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn(None, gt, w_in, t, consts)["line_of_sight_my"].backward()
    torch.cuda.current_stream().wait_stream(side)
    w_in.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        value = fn(None, gt, w_in, t, consts)["line_of_sight_my"]
        grad, = torch.autograd.grad(value, w_in)
    for eps, decay in ((5.5, 1.0), (4.0, 0.5), (2.5, 0.125)):
        consts.copy_(torch.tensor(loss.line_of_sight_consts(eps, decay)), non_blocking=True)
        graph.replay()
        v_f, g_f = _float_call(w, t, gt, eps, decay)
        assert torch.equal(value, v_f) and torch.equal(grad, g_f), (eps, decay)


# ----------------------------------------------------------------------------- 2. one iteration from a snapshot
def _snapshot(s):
    params = [p.detach().clone() for m in [s.model] + s.props for p in m.parameters()]
    opt = [[(g.exp_avg.clone(), g.exp_avg_sq.clone(), g.hyper.clone(), g.grad.clone(), g.lr_host) for g in o._groups]
           for o in (s.opt, s.est.optimizer)]
    return dict(params=params, opt=opt, sched=[copy.deepcopy(s.sched.state_dict()),
                                               copy.deepcopy(s.est.scheduler.state_dict())],
                lrs=[[grp["lr"] for grp in o.param_groups] for o in (s.opt, s.est.optimizer)],
                req=cic.req_cell(s.req_fn).cell_contents, decay=s.decay,
                cpu=torch.get_rng_state(), cuda=torch.cuda.get_rng_state())


def _restore(s, snap):
    with torch.no_grad():
        for p, v in zip([p for m in [s.model] + s.props for p in m.parameters()], snap["params"]):
            p.copy_(v)
    for o, groups, lrs in zip((s.opt, s.est.optimizer), snap["opt"], snap["lrs"]):
        for g, (m1, m2, h, gr, lr_host) in zip(o._groups, groups):
            g.exp_avg.copy_(m1); g.exp_avg_sq.copy_(m2); g.hyper.copy_(h); g.grad.copy_(gr); g.lr_host = lr_host
        for grp, lr in zip(o.param_groups, lrs):
            grp["lr"] = lr
    s.sched.load_state_dict(snap["sched"][0])
    s.est.scheduler.load_state_dict(snap["sched"][1])
    cic.req_cell(s.req_fn).cell_contents = snap["req"]
    s.decay = snap["decay"]
    torch.set_rng_state(snap["cpu"])
    torch.cuda.set_rng_state(snap["cuda"])


def _state(s):
    torch.cuda.synchronize()
    return dict(params=torch.cat([p.detach().reshape(-1) for m in [s.model] + s.props for p in m.parameters()]),
                m1=torch.cat([g.exp_avg for o in (s.opt, s.est.optimizer) for g in o._groups]),
                m2=torch.cat([g.exp_avg_sq for o in (s.opt, s.est.optimizer) for g in o._groups]),
                steps=[float(g.hyper[0]) for o in (s.opt, s.est.optimizer) for g in o._groups],
                lrs=[[grp["lr"] for grp in o.param_groups] for o in (s.opt, s.est.optimizer)],
                cpu=torch.get_rng_state(), cuda=torch.cuda.get_rng_state())


PIXEL_KEYS = ("psnr", "total_pixel_loss", "rgb_loss_l2", "sky_loss_opacity_based", "feature_loss_l2",
              "dynamic_sparsity_loss", "shadow_sparsity_loss", "cycle_loss", "max_forward_flow_norm",
              "max_backward_flow_norm", "max_forward_pred_backward_flow_norm", "max_backward_pred_forward_flow_norm")


EAGER_RUNS = 12


def _eager_runs(s, snap, step):
    """EAGER_RUNS eager iterations from the snapshot, cycling through three kernel overlaps (weight gradients on their
    side stream, on the main stream, everything on a side stream): [(logged row, state)].

    The float atomics of the backward sum in an order that depends on how the kernels are scheduled, and where a
    gradient entry is the residue of a cancellation, Adam (eps = 1e-15) turns the last-bit difference into an update of
    a different size.  Repeated eager runs from one snapshot land in such alternative outcomes too (seen: two groups
    5.3e-4 apart in the parameters of flow_feat, each holding eager runs of every overlap and replays), so one eager
    pair does not measure the spread; these runs do."""
    from emernerf_b200 import _ops

    runs = []
    for r in range(EAGER_RUNS):
        _restore(s, snap)
        mode = r % 3
        ws = _ops.WGRAD_STREAM
        try:
            _ops.WGRAD_STREAM = mode != 1
            if mode == 2:
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    row = cic.reference_iteration(s, step)
                torch.cuda.current_stream().wait_stream(side)
            else:
                row = cic.reference_iteration(s, step)
        finally:
            _ops.WGRAD_STREAM = ws
        runs.append((row, _state(s)))
    return runs


@pytest.mark.parametrize("variant,branch", [("static", None), ("dynamic", None), ("flow", None), ("flow_feat", None),
                                            ("flow", "fused")])
def test_replayed_iteration_matches_eager_from_a_snapshot(variant, branch, monkeypatch):
    from emernerf_b200 import _ops

    if branch is not None:
        monkeypatch.setattr(_ops, "FLOW_BRANCH", branch)
    s = cic.make_setup(variant, start_iter=2, decay_steps=3)
    it = cic.captured(s)
    checked = 0
    for step in range(40):
        if checked == 2:
            break
        s.decay = it.los.decay_weight
        snap = _snapshot(s)
        n = len(it.events)
        it(step)
        got_row = it.drain()[0]
        kinds = [e[0] for e in it.events[n:]]
        if kinds != ["replay", "replay"]:
            continue
        got = _state(s)
        after = _snapshot(s)
        eager = _eager_runs(s, snap, step)
        want_row, want = eager[0]
        assert s.decay == it.los.decay_weight
        assert list(got_row) == list(want_row)
        for k, v in want_row.items():
            if k in PIXEL_KEYS or k in ("lr", "epsilon"):
                assert all(row[k] == v for row, _ in eager), (step, k)       # the forward is deterministic
                assert got_row[k] == v, (step, k, got_row[k], v)
            else:
                spread = max(abs(row[k] - v) for row, _ in eager)
                bound = max(1e-4 * max(abs(v), 1e-12), 2 * spread)
                assert abs(got_row[k] - v) <= bound, (step, k, got_row[k], v, bound)
        for k in ("params", "m1", "m2"):
            spread = max(rel_err(st[k], want[k]) for _, st in eager)
            bound = max(1e-4, 2 * spread)
            assert rel_err(got[k], want[k]) <= bound, (step, k, rel_err(got[k], want[k]), bound)
        assert got["steps"] == want["steps"] and got["lrs"] == want["lrs"]
        assert torch.equal(got["cpu"], want["cpu"]) and torch.equal(got["cuda"], want["cuda"])
        _restore(s, after)                      # continue from the replayed state
        s.decay = it.los.decay_weight
        checked += 1
    assert checked == 2, it.events


# ----------------------------------------------------------------------------- 3. a trajectory through every branch
def _eager_trajectory(variant, steps, refresh_at):
    s = cic.make_setup(variant)
    s.dataset.pixel_source.pixel_error_buffered = False
    rows = []
    for step in range(steps):
        if step == refresh_at:
            s.dataset.pixel_sampler.refresh_pixel_error_maps(s.model, s.est, s.props, s.cfg)
        rows.append(cic.reference_iteration(s, step))
    return rows, s


def test_trajectory_through_every_branch():
    from emernerf_b200 import _lib

    variant, steps, refresh_at = "dynamic", 60, 20
    torch.manual_seed(0)
    torch.cuda.manual_seed(0)
    eager_a, sa = _eager_trajectory(variant, steps, refresh_at)
    peak_eager = torch.cuda.max_memory_reserved()
    torch.manual_seed(0)
    torch.cuda.manual_seed(0)
    eager_b, _ = _eager_trajectory(variant, steps, refresh_at)
    cuda_eager = torch.cuda.get_rng_state()

    torch.manual_seed(0)
    torch.cuda.manual_seed(0)
    s = cic.make_setup(variant)
    it = cic.captured(s)
    los = s.cfg.supervision.depth.line_of_sight
    s.dataset.pixel_source.pixel_error_buffered = False
    sa_decay = []
    rows = []
    for step in range(steps):
        if step == refresh_at:
            old = s.dataset.pixel_source.pixel_error_maps
            s.dataset.pixel_sampler.refresh_pixel_error_maps(s.model, s.est, s.props, s.cfg)
            assert s.dataset.pixel_source.pixel_error_maps is not old
        keys_before = {k: g.runs for k, g in it._graphs.items()}
        n_ev, n_launch = len(it.events), _lib.LAUNCHES
        torch.cuda.set_sync_debug_mode("warn")
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            it(step)
        torch.cuda.set_sync_debug_mode(0)
        new = it.events[n_ev:]
        if all(e[0] == "replay" for e in new):
            assert all(keys_before.get(e[1], 0) >= 2 for e in new)
            syncs = [w for w in caught if "synchroniz" in str(w.message).lower()]
            assert not syncs, (step, [str(w.message) for w in syncs])
            assert _lib.LAUNCHES == n_launch, step
        sa_decay.append(it.los.decay_weight)
        if step % 7 == 6 or step == steps - 1:
            rows.extend(it.drain())
    torch.cuda.synchronize()
    assert torch.equal(torch.cuda.get_rng_state(), cuda_eager)

    # the key sequence: every key eager once, captured at its second occurrence and replayed for it, then replayed;
    # the refresh at step 20 turns importance sampling on, so the captured pixel graphs of the old map are dropped
    seq = {}
    for kind, key in it.events:
        if kind == "drop":
            assert key[0] == "pixel" and key[2][0] is None and "capture" in seq[key]
            continue
        seq.setdefault(key, []).append(kind)
    for key, kinds in seq.items():
        runs = len(kinds) - ("capture" in kinds)
        assert kinds == (["eager"] + (["capture"] if runs > 1 else []) + ["replay"] * (runs - 1)), (key, kinds)
    assert any(e[0] == "drop" for e in it.events)
    req = cic.make_req_fn()
    want = set()
    for step in range(steps):
        want.add(("pixel", (req(step), step >= refresh_at)))
        want.add(("lidar", (req(step), step > los.start_iter)))
    assert {(k[0], k[1]) for k in seq} == want

    # host values exactly; device values within the spread of two eager runs
    assert len(rows) == steps
    decay = 1.0
    for step, (got, a, b) in enumerate(zip(rows, eager_a, eager_b)):
        if step > los.start_iter and (step - los.start_iter) % los.decay_steps == 0:
            decay *= los.decay_rate
        assert sa_decay[step] == decay
        assert list(got) == list(a), step
        assert got["lr"] == a["lr"] and got.get("epsilon") == a.get("epsilon"), step
        for k, v in a.items():
            if k in ("lr", "epsilon"):
                continue
            spread = max(abs(r[k] - e[k]) for r, e in zip(eager_a, eager_b) if k in r)
            tol = 4 * spread + 1e-5 * max(abs(v), 1.0)
            assert abs(got[k] - v) <= tol or (math.isnan(got[k]) and math.isnan(v)), (step, k, got[k], v, tol)

    # 4. one pool for every graph; the memory is reported, the pool asserted
    reserved = torch.cuda.memory_reserved()
    print(f"\n# eager peak reserved {peak_eager / 2**20:.0f} MiB, after capturing "
          f"{sum(g.graph is not None for g in it._graphs.values())} live graphs {reserved / 2**20:.0f} MiB")
    assert it._pool is not None
    assert all(g.graph.pool() == it._pool for g in it._graphs.values() if g.graph is not None)
