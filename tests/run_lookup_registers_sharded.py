#!/usr/bin/env python3
"""torchrun worker: proofs whose aux traces carry register columns (version-2 lookup programs, tests/test_lookup_registers.py),
split over WORLD_SIZE ranks (mdn_session_set_shard), must equal the unsplit proof, with the constraint guard off and on.
The LogUp and register build stays replicated: every rank builds the whole aux trace from its whole raw main trace.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/run_lookup_registers_sharded.py

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
    import test_lookup_registers as T
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    single, split = B.Session(params, local), B.Session(params, local)
    split.set_shard(rank, world, pkg.parallel.make_allgather_callback(dev_name))
    for name, case in (("chiplets 2^6 / 2^8", T.Case(6, 8)), ("chiplets 2^8 / 2^7", T.Case(8, 7)),
                       ("3 registers 2^9", T.KCase(3, 9)), ("4 registers 2^7", T.KCase(4, 7))):
        wl = case.wl(True)
        want = single.prove(wl.statement, wl.matrices, ch)
        for guard in (False, True):
            split.set_constraint_guard(guard)
            got = split.prove(wl.statement, wl.matrices, ch)
            assert same(got, want), f"rank {rank}: {name}, guard {guard}: the split proof differs from the unsplit proof"
        split.set_constraint_guard(False)
        if rank == 0:
            print(f"  ok: {name}", flush=True)
    split.close(); single.close()
    dist.barrier()
    print(f"LOOKUP_REGISTERS_SHARDED_OK rank={rank} world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
