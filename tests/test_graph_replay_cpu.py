"""The case lists and schedules of test_gpu_graph_replay.py, checked without a GPU: every bench workload is covered, the
training cases step as the bench does, and every schedule replays again after its eager interlude."""
import bench
from harness import train as H
from tests import test_gpu_graph_replay as G


def test_cases_cover_every_bench_workload():
    names = [c["name"] for c in G.QAT_CASES + G.PTQ_CASES]
    assert sorted(names) == sorted(H.WORKLOADS)
    assert len(names) == len(set(names))
    assert sorted(G.BENCH_ORDER) == sorted(H.WORKLOADS) and G.BENCH_ORDER[0] == bench.WORKLOAD


def test_qat_cases_step_like_the_bench():
    assert G.QAT_CASES
    for c in G.QAT_CASES:
        assert not H.WORKLOADS[c["name"]].get("inference")
        assert c["batch"] == bench.batch_per_gpu(c["name"]) == 256
        assert c["flat"] is True
        assert c["graph_warmup"] == 3 == H.QatStepper.__init__.__defaults__[-1]
    for c in G.PTQ_CASES:
        assert c["batch"] == bench.batch_per_gpu(c["name"])


def _phases(schedule):
    return [p for p, _ in schedule]


def test_schedules_replay_after_the_eager_interlude():
    for schedule, cap in ((G.SCHEDULE, G.GRAPH_WARMUP), (G.SCHEDULE, G.INFER_CAPTURE_STEP),
                          (G.SHORT_SCHEDULE + G.REVISIT, G.GRAPH_WARMUP),
                          (G.SHORT_SCHEDULE + G.REVISIT, G.INFER_CAPTURE_STEP)):
        rep = G.expected_replays(schedule, cap)
        ph = _phases(schedule)
        assert ph.count("eager") == 1 and "e2e" in ph
        first_eager = sum(n for p, n in schedule[:ph.index("eager")])
        after = first_eager + dict(schedule)["eager"]
        # warm-up as the bench runs it: at least 2 replays before the timed steps
        assert schedule[0] == ("resident", 5) and sum(rep[:5]) >= 2
        assert any(rep[cap + 1:first_eager]), "replays before the interlude"
        assert not any(rep[first_eager:after])
        assert any(rep[after:]), "no replay after the eager interlude"
    # consecutive steps see different batches, so a replay that kept its captured input shows at once
    assert G.NBUF == 4 and sum(n for _, n in G.SCHEDULE) > G.NBUF
