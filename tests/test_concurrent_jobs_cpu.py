"""TEST.CONCURRENT_JOBS on the host: the job split of imdb_detection_wrapper / imdb_proposal_extraction_wrapper, the
merge in job order, and the job-per-rank path on a gloo world of two.  The per-job pipelines are replaced by seeded
stubs whose output per image depends on the image alone, as the real pipeline's does (per-image soft-NMS, cut and
chips), so a correct split and merge reproduces the stub's per-image arrays in image order."""
import math
import os
import pickle
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sniper_b200 import iterator as IT  # noqa: E402
from sniper_b200 import tester as TS  # noqa: E402

K = 4
NET = SimpleNamespace(feat_stride=16, device="cpu")


def _roidb(n, salt=0):
    return [dict(image="im%03d.jpg" % i, width=100 + i + salt, height=80 + 3 * i, id=i) for i in range(n)]


def _boxes(r, c):
    rng = np.random.RandomState(r['id'] * 131 + c)
    return rng.rand(rng.randint(0, 5), 5).astype(np.float32)


def _props(r):
    rng = np.random.RandomState(7000 + r['id'])
    return rng.rand(rng.randint(1, 9), 5).astype(np.float32)


class _Stub(object):
    """Stands for tester._detection_job / _proposal_job: records every block it is given."""

    def __init__(self, fail_on_rank=None):
        self.blocks, self.fail_on_rank = [], fail_on_rank

    def _check(self, roidb):
        self.blocks.append([r['id'] for r in roidb])
        if self.fail_on_rank is not None and dist.is_initialized() and dist.get_rank() == self.fail_on_rank:
            raise RuntimeError("detect_post: the run buffer is full (stub)")

    def detection(self, net, config, roidb, num_classes, *args):
        self._check(roidb)
        assert num_classes == K and all(np.array_equal(r['inference_crops'], [[0, 0, r['width'], r['height']]])
                                        for r in roidb)
        boxes = [[[] for _ in roidb]] + [[_boxes(r, c) for r in roidb] for c in range(1, K)]
        return boxes, dict(scales=[dict(chips=len(roidb))], nms_s=0.0)

    def proposal(self, net, config, roidb, *args):
        self._check(roidb)
        return [_props(r) for r in roidb], dict(scales=[dict(images=len(roidb))])


class _Imdb(object):
    def evaluate_detections(self, all_boxes):
        return "eval of %d images" % len(all_boxes[1])

    def evaluate_recall(self, roidb, candidate_boxes=None):
        return "recall of %d images" % len(candidate_boxes)


def _cfg():
    cfg = IT.default_config()
    cfg.dataset.test_image_set = "stub"
    return cfg


def _detect(db, jobs, group=None):
    return TS.imdb_detection_wrapper(NET, _cfg(), db, num_classes=K, device="cpu", imdb=_Imdb(), concurrent_jobs=jobs,
                                     group=group)


def _extract(db, jobs, path, group=None):
    return TS.imdb_proposal_extraction_wrapper(NET, _cfg(), db, path, device="cpu", imdb=_Imdb(), concurrent_jobs=jobs,
                                               group=group)


def _want_boxes(db):
    return [[[] for _ in db]] + [[_boxes(r, c) for r in db] for c in range(1, K)]


def _same_boxes(a, b):
    return len(a) == len(b) and all(len(x) == len(y) and all(np.asarray(u).tobytes() == np.asarray(v).tobytes()
                                                             for u, v in zip(x, y)) for x, y in zip(a, b))


def test_job_blocks_are_the_reference_split():
    for n in range(61):
        for jobs in range(1, 10):
            per = int(math.ceil(float(n) / jobs))
            want = [[j for j in range(per * i, min(per * (i + 1), n))] for i in range(jobs)]
            got = TS.job_blocks(n, jobs)
            assert [list(range(lo, hi)) for lo, hi in got] == want, (n, jobs)
            assert all(0 <= lo <= hi <= n for lo, hi in got)
    assert [hi - lo for lo, hi in TS.job_blocks(5, 4)] == [2, 2, 1, 0]
    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError):
            TS.job_blocks(5, bad)


def test_one_job_calls_the_single_job_pipeline_unchanged(monkeypatch, tmp_path):
    db = _roidb(7)
    seen = []
    sentinel = ([[], []], dict(scales=["s"], nms_s=1.0))

    def job(net, config, roidb, *args):
        seen.append(roidb)
        return sentinel
    monkeypatch.setattr(TS, "_detection_job", job)
    boxes, stats = _detect(db, 1)
    assert len(seen) == 1 and seen[0] is db and boxes is sentinel[0] and stats is sentinel[1]
    assert set(stats) == {"scales", "nms_s", "eval", "eval_s"}
    stub = _Stub()
    monkeypatch.setattr(TS, "_proposal_job", stub.proposal)
    props, stats = _extract(db, 1, str(tmp_path))
    assert stub.blocks == [list(range(7))] and set(stats) == {"scales", "recall", "recall_s"}


@pytest.mark.parametrize("n,jobs", [(7, 2), (7, 3), (5, 4), (3, 5), (0, 2), (9, 9)])
def test_jobs_merge_in_job_order(monkeypatch, tmp_path, n, jobs):
    db = _roidb(n)
    stub = _Stub()
    monkeypatch.setattr(TS, "_detection_job", stub.detection)
    monkeypatch.setattr(TS, "_proposal_job", stub.proposal)
    blocks = [list(range(lo, hi)) for lo, hi in TS.job_blocks(n, jobs)]
    boxes, stats = _detect(db, jobs)
    assert stub.blocks == [b for b in blocks if b]                    # an empty job runs nothing
    assert _same_boxes(boxes, _want_boxes(db))
    assert stats["eval"] == "eval of %d images" % n and "scales" not in stats
    assert [(st["images"], st["rank"]) for st in stats["jobs"]] == [(b, 0) for b in TS.job_blocks(n, jobs)]
    assert [st["scales"] for st in stats["jobs"]] == [[dict(chips=len(b))] if b else [] for b in blocks]
    stub.blocks = []
    props, stats = _extract(db, jobs, str(tmp_path))
    assert stub.blocks == [b for b in blocks if b]
    want = [_props(r) for r in db]
    assert len(props) == n and all(a.tobytes() == b.tobytes() for a, b in zip(props, want))
    with open(os.path.join(str(tmp_path), TS.proposal_file_name(_cfg())), "rb") as f:
        saved = pickle.load(f)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(saved, want)) and len(saved) == n
    assert stats["recall"] == "recall of %d images" % n


# ---------------------------------------------------------------- two gloo ranks
def _rank(rank, port, case, tmp, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        stub = _Stub(fail_on_rank=1 if case == "fail" else None)
        TS._detection_job, TS._proposal_job = stub.detection, stub.proposal
        g = dist.group.WORLD
        if case in ("fail", "roidb"):
            db = _roidb(6, salt=rank if case == "roidb" else 0)
            try:
                _detect(db, 2, g)
                q.put((rank, "no error"))
            except Exception as e:
                q.put((rank, "%s: %s" % (type(e).__name__, e)))
            return
        out = []
        for n, jobs in ((7, 2), (7, 3), (5, 4), (1, 3), (0, 2)):
            db = _roidb(n)
            path = os.path.join(tmp, "%s_%d_%d_rank%d" % (case, n, jobs, rank))
            stub.blocks = []
            boxes, stats = _detect(db, jobs, g)
            props, pstats = _extract(db, jobs, path, g)
            mine = [j for j in range(jobs) if j % 2 == rank]
            listed = range(jobs) if rank == 0 else mine
            # a rank ran its own jobs alone, once for the detections and once for the proposals
            own = [list(range(*TS.job_blocks(n, jobs)[j])) for j in mine]
            checks = dict(ranks=[st["rank"] for st in stats["jobs"]] == [j % 2 for j in listed],
                          images=[st["images"] for st in pstats["jobs"]] == [TS.job_blocks(n, jobs)[j] for j in listed],
                          blocks=stub.blocks == [b for b in own if b] * 2)
            if rank == 0:
                one_boxes, _ = _detect(_roidb(n), jobs)
                one_props, _ = _extract(_roidb(n), jobs, path + "_one")
                name = TS.proposal_file_name(_cfg())
                checks.update(boxes=_same_boxes(boxes, one_boxes) and _same_boxes(boxes, _want_boxes(db)),
                              props=_same_boxes([props], [one_props]),
                              pickle=open(os.path.join(path, name), "rb").read() ==
                              open(os.path.join(path + "_one", name), "rb").read(),
                              eval=stats["eval"] == "eval of %d images" % n,
                              recall=pstats["recall"] == "recall of %d images" % n)
            else:
                checks.update(none=boxes is None and props is None, no_file=not os.path.exists(path),
                              no_eval="eval" not in stats and "recall" not in pstats)
            out.append(sorted(k for k, v in checks.items() if not v))
            dist.barrier()
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def _run_ranks(case, port, tmp):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, port, case, tmp, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        return dict(q.get(timeout=120) for _ in procs)
    finally:
        for p in procs:
            p.join(30)
            if p.is_alive():
                p.terminate()


def test_two_gloo_ranks_give_rank0_the_one_process_result(tmp_path):
    got = _run_ranks("merge", 29641, str(tmp_path))
    assert got == {0: [[]] * 5, 1: [[]] * 5}


def test_a_failing_job_raises_on_every_rank(tmp_path):
    got = _run_ranks("fail", 29643, str(tmp_path))
    for r in (0, 1):
        assert got[r].startswith("RuntimeError: concurrent test job 1 (images 3:6) failed on rank 1: RuntimeError: "
                                 "detect_post: the run buffer is full (stub)"), got


def test_mismatched_roidbs_raise_on_every_rank(tmp_path):
    got = _run_ranks("roidb", 29645, str(tmp_path))
    for r in (0, 1):
        assert got[r].startswith("ValueError: the ranks' test roidbs and concurrent_jobs differ"), got
