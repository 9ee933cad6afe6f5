"""TEST.CONCURRENT_JOBS on the device.

In one process: imdb_detection_wrapper / imdb_proposal_extraction_wrapper with concurrent_jobs=2 are byte-equal to
the per-image concatenation of two concurrent_jobs=1 calls on the two image blocks (AutoFocus pyramid, both detection
backends).  On two ranks: tools/test_e2e.py under torch.distributed.run (tests/concurrent_jobs_worker.py) on the
synthetic VOCdevkit from a checkpoint of a seeded network gives rank 0 the one-process J = 2 run's all_boxes,
do_python_eval text, proposal pickle bytes and recall string, and rank 1 writes no file.  On one GPU both ranks share
it over gloo (a correctness check only, not a speed); with two GPUs the script's own NCCL path runs, one GPU per rank."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import test_tester_gpu as TG  # noqa: E402
import train_data_fixture as TD  # noqa: E402
from sniper_b200 import checkpoint, model, synth_batch  # noqa: E402
from sniper_b200 import tester as TS  # noqa: E402

pytestmark = pytest.mark.gpu
WORKER = os.path.join(HERE, "concurrent_jobs_worker.py")


def _bytes_equal(a, b):
    return len(a) == len(b) and all(np.asarray(x).tobytes() == np.asarray(y).tobytes() and
                                    np.asarray(x).shape == np.asarray(y).shape for x, y in zip(a, b))


@pytest.fixture(scope="module")
def af_net():
    mc = model.Cfg()
    mc.batch_images = 2
    net = model.SniperResNet101(mc, deform_offset_std=0.01)
    net.train_step(synth_batch.make_batch(2, seed=7, device="cuda"), lr=0.001)      # non-trivial moving statistics
    net.enable_autofocus(seed=3)
    return net


def _db():
    rng = np.random.RandomState(11)
    return [dict(width=W, height=H, image_data=rng.randint(0, 256, (H, W, 3)).astype(np.uint8))
            for (W, H) in ((320, 240), (240, 320), (300, 200), (200, 260), (280, 280))]


@pytest.mark.parametrize("backend", ["device", "host"])
def test_two_jobs_equal_two_one_job_calls(af_net, tmp_path, backend):
    cfg = TG._small_cfg()
    db = _db()
    (lo0, hi0), (lo1, hi1) = TS.job_blocks(len(db), 2)
    assert (lo0, hi0, lo1, hi1) == (0, 3, 3, 5)
    both, stats = TS.imdb_detection_wrapper(af_net, cfg, db, detect_backend=backend, concurrent_jobs=2)
    chips = [np.array(r['inference_crops'], copy=True) for r in db]
    one = [TS.imdb_detection_wrapper(af_net, cfg, db[lo:hi], detect_backend=backend)[0] for lo, hi in ((0, 3), (3, 5))]
    assert [st["images"] for st in stats["jobs"]] == [(0, 3), (3, 5)] and all(len(st["scales"]) == 3
                                                                             for st in stats["jobs"])
    assert sum(st["scales"][0]["chips"] for st in stats["jobs"]) == 5
    for c in range(1, 81):
        assert _bytes_equal(both[c], one[0][c] + one[1][c]), c
    assert sum(len(d) for c in range(1, 81) for d in both[c]) > 0
    # the FocusChips of every image are the same whichever block it ran in
    assert all(np.array_equal(a, np.asarray(r['inference_crops'])) for a, r in zip(chips, db))
    if backend == "host":
        return
    cfg.dataset.test_image_set = "jobs"
    p2, _ = TS.imdb_proposal_extraction_wrapper(af_net, cfg, db, str(tmp_path / "j2"), concurrent_jobs=2)
    p1 = [TS.imdb_proposal_extraction_wrapper(af_net, cfg, db[lo:hi], str(tmp_path / ("j1_%d" % lo)))[0]
          for lo, hi in ((0, 3), (3, 5))]
    assert _bytes_equal(p2, p1[0] + p1[1]) and all(len(p) > 0 for p in p2)


# ---------------------------------------------------------------- tools/test_e2e.py on two ranks
@pytest.fixture(scope="module")
def voc(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("voc"))
    dk, _ = TD.write_voc(root, sets=(('2007', 'test', 5), ('2007', 'trainval', 3)), seed=4)
    mc = model.Cfg()
    mc.num_classes, mc.batch_images = 21, 1
    net = model.SniperResNet101(mc, device="cuda:0", seed=13)
    os.makedirs(os.path.join(root, "ckpt"))
    checkpoint.save_checkpoint(os.path.join(root, "ckpt", "seeded"), 1, *net.export_reference())
    del net
    torch.cuda.empty_cache()
    return root, dk


def _argv(voc, run, extract):
    root, dk = voc
    os.makedirs(os.path.join(run, "ckpt"), exist_ok=True)
    dst = os.path.join(run, "ckpt", "seeded-0001.params")
    if not os.path.exists(dst):
        os.link(os.path.join(root, "ckpt", "seeded-0001.params"), dst)
    argv = ["--dataset", "PascalVOC", "--root-path", root, "--dataset-path", dk, "--prefix",
            os.path.join(run, "ckpt", "seeded"), "--epoch", "1", "--network", "resnet101"]
    if extract:
        argv += ["--extract-proposals", "--image-set", "2007_test+2007_trainval", "--proposal-save-path",
                 os.path.join(run, "proposals")]
    else:
        argv += ["--image-set", "2007_test"]
    return argv


def _run(cmd, out, name):
    os.makedirs(out, exist_ok=True)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=dict(os.environ, OMP_NUM_THREADS="4"),
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    with open(os.path.join(out, name + ".pkl"), "rb") as f:
        return pickle.load(f)


def _one_process(voc, tmp_path, extract):
    run = str(tmp_path / "one")
    argv = _argv(voc, run, extract) + ["--concurrent-jobs", "2", "--device", "cuda:0"]
    return _run([sys.executable, WORKER, "one", run] + argv, run, "one"), run


def _two_ranks(voc, tmp_path, extract, backend, port):
    run = str(tmp_path / "ranks")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), WORKER, "ranks", run, backend] + _argv(voc, run, extract)
    r0 = _run(cmd, run, "rank0")
    with open(os.path.join(run, "rank1.pkl"), "rb") as f:
        r1 = pickle.load(f)
    return r0, r1, run


def _check(voc, tmp_path, extract, backend, port):
    one, one_dir = _one_process(voc, tmp_path, extract)
    r0, r1, ranks_dir = _two_ranks(voc, tmp_path, extract, backend, port)
    assert (one["world"], r0["rank"], r0["world"], r1["rank"], r1["world"]) == (1, 0, 2, 1, 2)
    assert r1["written"] == [] and r0["written"]
    sets = ["2007_test", "2007_trainval"] if extract else ["2007_test"]
    assert sorted(one["results"]) == sorted(r0["results"]) == sorted(r1["results"]) == sorted(sets)
    for s in sets:
        (want, want_st), (got, got_st) = one["results"][s], r0["results"][s]
        assert r1["results"][s][0] is None and r1["results"][s][1] == {}
        if extract:
            assert _bytes_equal(got, want) and sum(len(p) for p in got) > 0
            name = "PASCALVOC_%s_rpn.pkl" % s
            a = open(os.path.join(one_dir, "proposals", name), "rb").read()
            b = open(os.path.join(ranks_dir, "proposals", name), "rb").read()
            assert a == b
            assert got_st["recall"] == want_st["recall"] and got_st["recall"]
        else:
            assert len(got) == 21 and all(_bytes_equal(g, w) for g, w in zip(got, want))
            assert got_st["eval"] == want_st["eval"] and got_st["eval"].startswith("VOC07 metric?")


@pytest.mark.parametrize("extract", [False, True], ids=["detect", "proposals"])
def test_two_ranks_on_one_gpu_gloo(voc, tmp_path, extract):
    _check(voc, tmp_path, extract, "gloo", 29551 + extract)


@pytest.mark.parametrize("extract", [False, True], ids=["detect", "proposals"])
def test_two_ranks_on_two_gpus_nccl(voc, tmp_path, extract):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _check(voc, tmp_path, extract, "nccl", 29555 + extract)
