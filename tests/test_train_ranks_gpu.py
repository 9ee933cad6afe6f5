"""Data-parallel training from an image set on disk: tools/train_e2e.py's main on two ranks (tests/ranks_worker.py under
torch.distributed.run) over the synthetic VOCdevkit, two chips per rank, two epochs.

On one GPU both ranks share it over gloo (a correctness check only, not a speed); with two GPUs the launcher's own NCCL
path runs, one GPU per rank.  Checked after every epoch: (a) both ranks hold byte-identical weights and momenta;
(b) rank 0 alone writes each `.params` / `.states` file; (c) the weights and momenta are byte-equal to a one-process
emulation (two networks, each on one rank's slice, gradients summed g0 + g1, one update each) and the checkpoint's
BatchNorm moving statistics are byte-equal to (m0 + m1) / 2 of the emulation's two networks; (d) on one GPU, a run
resumed from the epoch-1 checkpoint ends with the weights and momenta of the uninterrupted run."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import train_data_fixture as TD  # noqa: E402
from sniper_b200 import checkpoint  # noqa: E402

pytestmark = pytest.mark.gpu
WORKER = os.path.join(HERE, "ranks_worker.py")
EPOCHS = 2


def _argv(root, dk, prefix, *extra):
    return ["--dataset", "PascalVOC", "--image-set", "2007_trainval+2012_trainval", "--root-path", root,
            "--dataset-path", dk, "--batch-size", "2", "--display", "2", "--prefix", prefix, "--epochs", str(EPOCHS),
            "--seed", "3"] + list(extra)


def _launch(out, backend, argv, port):
    os.makedirs(out, exist_ok=True)
    env = dict(os.environ, OMP_NUM_THREADS="4")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), WORKER, "train", out, backend] + argv
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    return [json.load(open(os.path.join(out, "rank%d.json" % k))) for k in range(2)]


def _emulate(out, argv):
    os.makedirs(out, exist_ok=True)
    r = subprocess.run([sys.executable, WORKER, "emulate", out] + argv, capture_output=True, text=True, timeout=1200,
                       cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]


def _npz(path):
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


def _aux(d):
    return {k[4:]: v for k, v in d.items() if k.startswith("aux:")}


def _same(a, b, keys=("w", "mom")):
    return {k: a[k].tobytes() == b[k].tobytes() for k in keys}


def _check_run(run, emul, prefix, ranks):
    # (b) rank 0 alone wrote the checkpoints, and they are all there
    assert [r["rank"] for r in ranks] == [0, 1] and all(r["world"] == 2 for r in ranks)
    assert ranks[0]["written"] == list(range(1, EPOCHS + 1)) and ranks[1]["written"] == []
    assert ranks[0]["num_update"] == ranks[1]["num_update"] > 0
    for ep in range(1, EPOCHS + 1):
        assert os.path.isfile("%s-%04d.params" % (prefix, ep)) and os.path.isfile("%s-%04d.states" % (prefix, ep))
        r0, r1 = (_npz(os.path.join(run, "rank%d_ep%d.npz" % (k, ep))) for k in range(2))
        e0, e1 = (_npz(os.path.join(emul, "emul%d_ep%d.npz" % (k, ep))) for k in range(2))
        # (a) the ranks agree
        assert _same(r0, r1) == {"w": True, "mom": True}, ep
        # (c) the emulation agrees, and its two networks with each other
        assert _same(e0, e1) == {"w": True, "mom": True}, ep
        assert _same(r0, e0) == {"w": True, "mom": True}, ep
        arg, aux = checkpoint.load_param(prefix, ep)
        a0, a1 = _aux(e0), _aux(e1)
        assert set(aux) == set(a0)
        bad = [k for k in aux if aux[k].tobytes() != ((a0[k] + a1[k]) / np.float32(2)).tobytes()]
        assert not bad, (ep, bad[:5])
        # the per-rank statistics of the run itself are the emulation's: each rank kept its own
        assert all(_aux(r0)[k].tobytes() == a0[k].tobytes() and _aux(r1)[k].tobytes() == a1[k].tobytes() for k in a0)
        # the per-rank statistics differ somewhere (each rank saw its own chips), so the average is not a no-op
        assert any(a0[k].tobytes() != a1[k].tobytes() for k in a0)
    assert json.load(open(os.path.join(emul, "emul.json")))["steps"] == ranks[0]["num_update"]


@pytest.fixture(scope="module")
def voc(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("voc"))
    dk, _ = TD.write_voc(root)
    return root, dk


@pytest.mark.parametrize("bf16", [False, True], ids=["tf32", "bf16"])
def test_two_ranks_on_one_gpu_gloo(voc, tmp_path, bf16):
    root, dk = voc
    extra = ["--bf16"] if bf16 else []
    prefix = str(tmp_path / "out" / "voc")
    ranks = _launch(str(tmp_path / "run"), "gloo", _argv(root, dk, prefix, *extra), 29531 + bf16)
    _emulate(str(tmp_path / "emul"), _argv(root, dk, str(tmp_path / "emul_out" / "voc"), *extra))
    _check_run(str(tmp_path / "run"), str(tmp_path / "emul"), prefix, ranks)
    if bf16:
        return
    # (d) resumed from the epoch-1 checkpoint (every rank loads the same files): the same weights and momenta at the
    # end; the .states file (momenta and update count) byte-equal
    res_prefix = str(tmp_path / "resumed" / "voc")
    os.makedirs(os.path.dirname(res_prefix))
    for ext in ("params", "states"):
        shutil.copy("%s-0001.%s" % (prefix, ext), "%s-0001.%s" % (res_prefix, ext))
    ranks_r = _launch(str(tmp_path / "run_r"), "gloo", _argv(root, dk, res_prefix, "--begin-epoch", "1"), 29535)
    assert ranks_r[0]["written"] == [EPOCHS] and ranks_r[1]["written"] == []
    assert ranks_r[0]["num_update"] == ranks[0]["num_update"]
    for k in range(2):
        a = _npz(os.path.join(str(tmp_path / "run"), "rank%d_ep%d.npz" % (k, EPOCHS)))
        b = _npz(os.path.join(str(tmp_path / "run_r"), "rank%d_ep%d.npz" % (k, EPOCHS)))
        assert _same(a, b) == {"w": True, "mom": True}, k
    arg, aux = checkpoint.load_param(prefix, EPOCHS)
    arg_r, aux_r = checkpoint.load_param(res_prefix, EPOCHS)
    assert all(arg[k].tobytes() == arg_r[k].tobytes() for k in arg)
    assert open("%s-%04d.states" % (prefix, EPOCHS), "rb").read() == open("%s-%04d.states" % (res_prefix, EPOCHS),
                                                                           "rb").read()
    # the moving statistics: every rank resumed from the averaged ones (as a reloaded reference checkpoint does), so
    # they continue from a different start than the uninterrupted run's per-rank values; they stay close
    for k in aux:
        assert np.allclose(aux[k], aux_r[k], rtol=1e-4, atol=1e-5), k


def test_two_ranks_on_two_gpus_nccl(voc, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root, dk = voc
    prefix = str(tmp_path / "out" / "voc")
    ranks = _launch(str(tmp_path / "run"), "nccl", _argv(root, dk, prefix), 29537)
    _emulate(str(tmp_path / "emul"), _argv(root, dk, str(tmp_path / "emul_out" / "voc"), "--device", "cuda:0"))
    _check_run(str(tmp_path / "run"), str(tmp_path / "emul"), prefix, ranks)
