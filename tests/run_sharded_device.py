#!/usr/bin/env python3
"""torchrun worker: ONE proof split over WORLD_SIZE ranks from column-major device traces (MDN_FLAG_DEVICE_TRACES |
MDN_FLAG_COLUMN_MAJOR, every rank ingesting its own whole copy) with a device aux builder must be byte-identical to the
unsplit proof of the same statement from host row-major traces with the equivalent host builder.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/run_sharded_device.py

On the CPU kernel emulator (MDN_ALLOW_EMULATOR=1 MDN_EMU_SHM=1) device memory is host memory and gloo carries the
bootstrap, as in tests/run_sharded.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import pkgload

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    if os.environ.get("MDN_ALLOW_EMULATOR") == "1":
        dist.init_process_group("gloo")
        local, dev_name = 0, "cpu"
    else:
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        dev_name = f"cuda:{local}"
    import test_airs as TA
    import test_device_resident as D
    params = W.fast_pcs_params()
    cases = [("dummy AIRs, device aux builder", D.dummy_case([9, 7], (9, 10), (1, 2))),
             ("fib + dummy, device aux builder", TA.fib_product_workload([8, 6], lqd=1)),
             ("LogUp read from the caller's trace", (TA.logup_workload(7, device=True)[0], None))]
    ref_sess = B.Session(params, local)
    split = B.Session(params, local)
    split.set_shard(rank, world, pkg.parallel.make_allgather_callback(dev_name))
    for name, (wl, builder) in cases:
        ch = D.TC.seed(params)
        ref = ref_sess.prove(wl.statement, wl.matrices, ch, B.AUX_BUILDER(builder) if builder else None)
        mats, bufs = D.column_major_traces(wl)
        split.set_device_aux_builder(D.device_builder(wl, builder, bufs))
        got = split.prove(wl.statement, mats, ch, None, D.CM)
        split.set_device_aux_builder(None)
        assert D.same(ref, got), f"rank {rank}: {name}: the split column-major proof differs from the unsplit host proof"
        print(f"rank {rank}: {name}: ok", flush=True)
    split.close()
    ref_sess.close()
    dist.barrier()
    if rank == 0:
        print(f"SHARDED_DEVICE_OK world={world}", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
