#!/usr/bin/env python3
"""torchrun worker: the constraint guard on a proof split over WORLD_SIZE ranks (mdn_session_set_shard).  Every rank
holds the whole raw main and aux traces and runs the whole check on them, so:
  * a statement that holds gets, with the guard on, the proof the unsplit session makes with the guard off;
  * a statement with one fault is refused on every rank with MDN_ERR_CONSTRAINT_VIOLATED and the report of the unsplit
    guarded session, and every rank proves the next valid statement again.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/run_guard_sharded.py

tests/test_constraint_guard_emulated.py runs it on the CPU kernel emulator (MDN_ALLOW_EMULATOR=1 MDN_EMU_SHM=1, gloo) at
worlds 2 and 4, as tests/run_sharded.py is run for the split proof."""
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


def report(rep):
    return (rep.holds, rep.kind, rep.instance, rep.constraint, rep.row, rep.value[0], rep.value[1], rep.failing_rows)


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
    import test_airs
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    single, split = B.Session(params, local), B.Session(params, local)
    split.set_shard(rank, world, pkg.parallel.make_allgather_callback(dev_name))
    split.set_constraint_guard(True)

    # statements that hold: host aux builder with a taller dummy AIR, device LogUp build, preprocessed columns
    wl, bld = test_airs.fib_product_workload([8, 9], lqd=1)
    cases = [("host aux builder", wl, bld), ("LogUp aux built on the device", test_airs.logup_workload(8, device=True)[0], None),
             ("preprocessed columns", test_airs.preprocessed_workload((7, 8), (True, True)), None)]
    for name, wl, bld in cases:
        for s in (single, split):
            if getattr(wl, "preprocessed", None) is not None:
                s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
            else:
                s.set_preprocessed(None, None)
        cb = B.AUX_BUILDER(bld) if bld is not None else None
        want = single.prove(wl.statement, wl.matrices, ch, cb)
        got = split.prove(wl.statement, wl.matrices, ch, cb)
        assert same(got, want), f"rank {rank}: case '{name}': the guarded split proof differs from the unsplit proof"
        assert split.last_constraint_report().holds == 1
    for s in (single, split):
        s.set_preprocessed(None, None)

    # one fault in the taller instance's trace (a transition, past every rank's first slice) and one in the host aux
    single.set_constraint_guard(True)
    for name, row, col in (("main cell", 300, 1), ("aux cell", None, None)):
        wl, bld = test_airs.fib_product_workload([9, 8], lqd=1)
        if row is not None:
            wl.traces[0][row, col] = (int(wl.traces[0][row, col]) + 1) % W.P
            cb = B.AUX_BUILDER(bld)
        else:
            def bad(ctx, inst, main, rnd, aux_out, aux_values, bld=bld):
                r = bld(ctx, inst, main, rnd, aux_out, aux_values)
                if inst == 0:
                    aux_out[2 * 411 + 1] = (aux_out[2 * 411 + 1] + 1) % W.P
                return r
            cb = B.AUX_BUILDER(bad)
        reps = []
        for s in (single, split):
            try:
                s.prove(wl.statement, wl.matrices, ch, cb)
                raise SystemExit(f"rank {rank}: case '{name}': a violating statement was proved")
            except B.ConstraintViolation as e:
                reps.append(report(e.report))
        assert reps[0] == reps[1] and reps[0][1] == 1, f"rank {rank}: case '{name}': {reps}"
        every = [None] * world
        dist.all_gather_object(every, reps[1])
        assert all(r == reps[1] for r in every), f"case '{name}': the ranks disagree: {every}"
        if rank == 0:
            print(f"  refused: {name}: {reps[1]}", flush=True)
    wl, bld = test_airs.fib_product_workload([8, 9], lqd=1)
    want = single.prove(wl.statement, wl.matrices, ch, B.AUX_BUILDER(bld))
    assert same(split.prove(wl.statement, wl.matrices, ch, B.AUX_BUILDER(bld)), want), f"rank {rank}: no proof after a refusal"
    split.close(); single.close()
    dist.barrier()
    print(f"GUARD_SHARDED_OK rank={rank} world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
