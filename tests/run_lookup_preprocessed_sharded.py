#!/usr/bin/env python3
"""torchrun worker: proofs whose LogUp aux traces read preprocessed columns (tests/test_lookup_preprocessed.py), split
over WORLD_SIZE ranks (mdn_session_set_shard), must equal the unsplit proof, with the constraint guard off and on.  The
LogUp build stays replicated: every rank derives the preprocessed rows from its whole copy of the bundle.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/run_lookup_preprocessed_sharded.py

On the CPU kernel emulator (MDN_ALLOW_EMULATOR=1 MDN_EMU_SHM=1) the ranks run over gloo, as in tests/run_sharded.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist
import pkgload

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding


def same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if os.environ.get("MDN_ALLOW_EMULATOR") == "1":
        dist.init_process_group("gloo")
        local, dev_name = 0, "cpu"
    else:
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        dev_name = f"cuda:{local}"
    import helpers as H
    import test_lookup_preprocessed as T
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    single, split = B.Session(params, local), B.Session(params, local)
    split.set_shard(rank, world, pkg.parallel.make_allgather_callback(dev_name))
    for heights in ((6, 8), (8, 7)):
        wl = T.Case(*heights).wl(True)
        for s in (single, split):
            s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
        want = single.prove(wl.statement, wl.matrices, ch)
        for guard in (False, True):
            split.set_constraint_guard(guard)
            got = split.prove(wl.statement, wl.matrices, ch)
            assert same(got, want), f"rank {rank}: heights {heights}, guard {guard}: the split proof differs from the unsplit proof"
        split.set_constraint_guard(False)
        if rank == 0:
            print(f"  ok: heights {heights}", flush=True)
    split.close(); single.close()
    dist.barrier()
    print(f"LOOKUP_PREP_SHARDED_OK rank={rank} world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
