"""Worker of tests/test_concurrent_jobs_gpu.py: tools/test_e2e.py's main, its results pickled to <out>/<name>.pkl.

    python tests/concurrent_jobs_worker.py one <out> <test_e2e args>
        one process (--concurrent-jobs in the args).
    python -m torch.distributed.run --nproc-per-node 2 tests/concurrent_jobs_worker.py ranks <out> gloo|nccl <args>
        every rank (gloo: joined here, both ranks on cuda:0; nccl: initialised by test_e2e on cuda:LOCAL_RANK); each
        rank also records the files it opened for writing during main."""
import builtins
import os
import pickle
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import test_e2e as T  # noqa: E402


def run(out, name, argv):
    written = []
    real_open = builtins.open

    def recording_open(file, mode="r", *a, **k):
        if any(c in mode for c in "wax+"):
            written.append(str(file))
        return real_open(file, mode, *a, **k)
    builtins.open = recording_open
    try:
        res = T.main(argv)
    finally:
        builtins.open = real_open
    results = {s: (boxes, {k: v for k, v in st.items() if k in ("eval", "recall")})
               for s, (boxes, st) in res["results"].items()}
    with open(os.path.join(out, name + ".pkl"), "wb") as f:
        pickle.dump(dict(rank=res["rank"], world=res["world_size"], results=results, written=written), f)


if __name__ == "__main__":
    mode, out = sys.argv[1], sys.argv[2]
    if mode == "one":
        run(out, "one", sys.argv[3:])
    else:
        import torch.distributed as dist
        backend, argv = sys.argv[3], sys.argv[4:]
        if backend == "gloo":
            dist.init_process_group("gloo")
            argv = argv + ["--device", "cuda:0"]
        run(out, "rank%s" % os.environ["RANK"], argv)
        if backend == "gloo":
            dist.destroy_process_group()
