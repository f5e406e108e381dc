"""The CUDA-graph replay of every bench workload's step against eager steps of the same model, bit for bit.

Every number bench.py reports comes from a replay: ``QatStepper(graph=True)`` captures forward + loss + zero_grad +
backward once after ``graph_warmup`` eager steps and replays it (FlatAdam runs outside the graph), ``InferStepper(graph=True)``
does the same for the PTQ forward.  A replay can compute something else while the throughput looks fine: Python-side state
frozen at capture time, a scratch buffer (re)allocated during or after capture, a gradient bucket not zeroed inside the
graph, static inputs not refreshed, eager steps between replays allocating from the non-graph pool.  The engine is
deterministic (fixed-order reductions), so a replayed trajectory must equal an eager one bit for bit.

The steppers are driven as bench.run_engine drives them (same batch size, 4 rotating seeded batches, resident and
pinned-host-fed steps, the graph switched off for an eager interlude and restored), without run_engine itself."""
import gc

import pytest
import torch

import bench
from harness import train as H

pytestmark = pytest.mark.gpu
NBUF = 4
GRAPH_WARMUP = 3            # QatStepper's default: the bench never sets it
INFER_CAPTURE_STEP = 2      # InferStepper captures at its third step

# the bench's schedule for one workload: (phase, steps).  "resident": batches already on the device; "e2e": pinned host
# batches copied non_blocking to the device (bench step_e2e); "eager": the graph switched off as the bench does it for its
# per-kernel detail pass (stepper.graph, stepper.graph_wanted = None, False); "restored": the saved graph put back
SCHEDULE = (("resident", 5), ("resident", 6), ("e2e", 2), ("eager", 3), ("restored", 2))
# the one-process test: shorter, and every stepper comes back for two more replays after the later workloads captured
SHORT_SCHEDULE = (("resident", 5), ("e2e", 1), ("eager", 2), ("restored", 1))
REVISIT = (("restored", 2),)

QAT_CASES = [dict(name=n, batch=bench.batch_per_gpu(n), flat=True, graph_warmup=GRAPH_WARMUP)
             for n, w in H.WORKLOADS.items() if not w.get("inference")]
PTQ_CASES = [dict(name=n, batch=bench.batch_per_gpu(n)) for n, w in H.WORKLOADS.items() if w.get("inference")]
# bench order: the headline workload first, then the others in WORKLOADS order
BENCH_ORDER = [bench.WORKLOAD] + [n for n in H.WORKLOADS if n != bench.WORKLOAD]


def expected_replays(schedule, capture_step):
    """per step of ``schedule``: True where a graph-wanting stepper replays (capture happens at ``capture_step``)"""
    out, k, on = [], 0, True
    for phase, n in schedule:
        if phase == "eager":
            on = False
        elif phase == "restored":
            on = True
        for _ in range(n):
            out.append(on and k >= capture_step)
            k += 1
    return out


def _bits(t):
    t = t.detach().contiguous().cpu()
    return t.reshape(-1).view(torch.uint8)


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _build(name, dev):
    w = H.WORKLOADS[name]
    return H.prepare_engine(H.build_float_model(w["model"]), w["scheme"], **w["prepare"],
                            **w.get("engine_extra", {})).to(dev)


def _batches(name, dev):
    w = H.WORKLOADS[name]
    host = [H.synthetic_batch(bench.batch_per_gpu(name), w["hw"], seed=100 + i, pin=True) for i in range(NBUF)]
    return host, [(x.to(dev), t.to(dev)) for x, t in host]


class Run:
    """one workload stepped through a schedule; keeps what each step computed (on the device until ``finish``)"""

    def __init__(self, name, graph, dev):
        from micronet_b200 import _lib as L
        self.L, self.name, self.dev, self.graph = L, name, dev, graph
        w = H.WORKLOADS[name]
        self.inference = bool(w.get("inference"))
        self.model = _build(name, dev)
        self.host, self.devb = _batches(name, dev)
        B = bench.batch_per_gpu(name)
        if self.inference:
            self.stepper = H.InferStepper(self.model, graph=graph)
            self.stepper.calibrate([self.devb[i][0][: max(2, B // 8)] for i in range(w.get("calib_batches", 2))])
        else:
            self.stepper = H.QatStepper(self.model, lr=0.01, wd=w["wd"], flat=True, graph=graph,
                                        graph_warmup=GRAPH_WARMUP)
        self.k, self.outs, self.launches, self.replayed, self.saved = 0, [], [], [], None
        self.capture_step = INFER_CAPTURE_STEP if self.inference else GRAPH_WARMUP

    def run(self, schedule):
        st = self.stepper
        for phase, n in schedule:
            if phase == "eager" and self.saved is None:
                self.saved = (st.graph, st.graph_wanted)
                st.graph, st.graph_wanted = None, False
            elif phase == "restored" and self.saved is not None:
                st.graph, st.graph_wanted = self.saved
                self.saved = None
            for _ in range(n):
                i = self.k % NBUF
                if phase == "e2e":
                    hx, ht = self.host[i]
                    x, t = hx.to(self.dev, non_blocking=True), ht.to(self.dev, non_blocking=True)
                else:
                    x, t = self.devb[i]
                n0 = self.L.launch_count()
                # detached at once: a live autograd graph would reach into the next capture.  Cloned: the next replay
                # overwrites static_loss / static_out
                out = st.step(x, t).detach().clone()
                self.launches.append(self.L.launch_count() - n0)
                self.replayed.append(st.graph is not None)
                self.outs.append(out)
                if self.graph and self.k == self.capture_step:
                    assert st.graph is not None and st.graph_error is None, (self.name, st.graph_error)
                self.k += 1
        return self

    def finish(self):
        """synchronise, check the tensor-core flag, move everything to the host and free the model"""
        torch.cuda.synchronize()
        self.L.tc_check()
        res = {"outs": [o.cpu() for o in self.outs], "launches": list(self.launches), "replayed": list(self.replayed),
               "graph_error": getattr(self.stepper, "graph_error", None), "state": {}}
        state = res["state"]
        for n, p in self.model.named_parameters():
            state["param " + n] = p.detach().cpu()
        for n, b in self.model.named_buffers():
            state["buffer " + n] = b.detach().cpu()
        if not self.inference:
            opt = self.stepper.opt
            state["adam exp_avg"] = opt.exp_avg.cpu()
            state["adam exp_avg_sq"] = opt.exp_avg_sq.cpu()
            state["grad bucket"] = opt.bucket.flat.cpu()
        del self.stepper, self.model, self.outs, self.devb
        self.saved = None
        gc.collect()
        torch.cuda.empty_cache()
        return res


def trajectory(name, graph, schedule):
    dev = torch.device("cuda", torch.cuda.current_device())
    return Run(name, graph, dev).run(schedule).finish()


def assert_same_trajectory(name, got, ref, what):
    """bitwise: every step's loss / logits, then every tensor of the final state"""
    assert len(got["outs"]) == len(ref["outs"])
    for k, (a, b) in enumerate(zip(got["outs"], ref["outs"])):
        if not _same_bits(a, b):
            d = (a.double() - b.double()).abs().max().item() if a.shape == b.shape else None
            raise AssertionError(f"{name}: step {k} ({what}) differs from the eager step, max |diff| {d}")
    assert got["state"].keys() == ref["state"].keys()
    bad = [n for n in ref["state"] if not _same_bits(got["state"][n], ref["state"][n])]
    assert not bad, f"{name}: after {len(ref['outs'])} steps ({what}) these differ from the eager run: {bad[:8]}"


def assert_replayed(name, res, schedule, capture_step):
    """the graph was used where it should be: no launch through the engine's wrappers on a replayed step but FlatAdam's"""
    want = expected_replays(schedule, capture_step)
    assert res["graph_error"] is None, (name, res["graph_error"])
    assert res["replayed"] == want, (name, res["replayed"], want)
    limit = 0 if H.WORKLOADS[name].get("inference") else 1
    for k, (rep, n) in enumerate(zip(want, res["launches"])):
        if k == capture_step:      # the capture runs the engine's wrappers once more, then replays
            continue
        if rep:
            assert n <= limit, f"{name}: replayed step {k} issued {n} engine launches"
        else:
            assert n >= 10, f"{name}: eager step {k} issued only {n} engine launches"


# ---------------------------------------------------------------------------------------------------------------------
# determinism precondition: two fresh eager trajectories are bitwise equal
# ---------------------------------------------------------------------------------------------------------------------
_EAGER = {}


def eager_reference(name):
    if name not in _EAGER:
        _EAGER[name] = trajectory(name, False, SCHEDULE)
    return _EAGER[name]


def _first_divergence(name, step):
    """two fresh eager runs up to ``step``; that step runs with hooks on every module: the first module (forward order)
    whose output differs, else the first (backward order) whose output gradient differs"""
    dev = torch.device("cuda", torch.cuda.current_device())
    recs = []
    for _ in range(2):
        r = Run(name, False, dev)
        r.run(((("resident", step),) if step else ()))
        fwd, bwd, hooks = [], [], []

        def fhook(mod, inp, out, mname=None):
            if isinstance(out, torch.Tensor):
                fwd.append((mname, out.detach().cpu()))
                if out.requires_grad:
                    out.register_hook(lambda g: bwd.append((mname, g.detach().cpu())))

        for mname, mod in r.model.named_modules():
            if mname:
                hooks.append(mod.register_forward_hook(lambda m, i, o, mname=mname: fhook(m, i, o, mname)))
        r.run((("resident", 1),))
        torch.cuda.synchronize()
        for h in hooks:
            h.remove()
        recs.append((fwd, bwd))
        r.finish()
    for kind, a, b in (("output", recs[0][0], recs[1][0]), ("output gradient", recs[0][1], recs[1][1])):
        for (ma, ta), (_, tb) in zip(a, b):
            if not _same_bits(ta, tb):
                return f"{kind} of module {ma!r}"
    return "no module output or gradient (the difference is in the optimizer or a buffer)"


@pytest.mark.parametrize("name", [c["name"] for c in QAT_CASES])
def test_eager_qat_step_is_deterministic(name):
    a = eager_reference(name)
    b = trajectory(name, False, SCHEDULE)
    for k, (x, y) in enumerate(zip(a["outs"], b["outs"])):
        if not _same_bits(x, y):
            raise AssertionError(f"{name}: two eager runs differ at step {k}; first at {_first_divergence(name, k)}")
    assert_same_trajectory(name, b, a, "two eager runs")


# ---------------------------------------------------------------------------------------------------------------------
# graph replay against eager
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c["name"] for c in QAT_CASES])
def test_qat_graph_replay_equals_eager_steps(name):
    ref = eager_reference(name)
    got = trajectory(name, True, SCHEDULE)
    assert_replayed(name, got, SCHEDULE, GRAPH_WARMUP)
    assert not any(ref["replayed"])
    assert_same_trajectory(name, got, ref, "graph replay")


@pytest.mark.parametrize("name", [c["name"] for c in PTQ_CASES])
def test_ptq_graph_replay_equals_eager_forward(name):
    ref = trajectory(name, False, SCHEDULE)
    got = trajectory(name, True, SCHEDULE)
    assert_replayed(name, got, SCHEDULE, INFER_CAPTURE_STEP)
    assert not any(ref["replayed"])
    assert_same_trajectory(name, got, ref, "graph replay")


def test_every_workload_in_bench_order_in_one_process():
    """the workloads share module-level caches (_lib._scratch / _errflags, pk._plan_cache, the DoReFa scale tensors): every
    stepper captures with the earlier workloads' graphs still alive, then each replays again after all have captured"""
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = [Run(name, True, dev).run(SHORT_SCHEDULE) for name in BENCH_ORDER]
    for r in runs:
        r.run(REVISIT)
    got = {r.name: r.finish() for r in runs}
    del runs
    for name in BENCH_ORDER:
        cap = INFER_CAPTURE_STEP if H.WORKLOADS[name].get("inference") else GRAPH_WARMUP
        assert_replayed(name, got[name], SHORT_SCHEDULE + REVISIT, cap)
        ref = trajectory(name, False, SHORT_SCHEDULE + REVISIT)
        assert_same_trajectory(name, got[name], ref, "graph replay, all workloads in one process")
