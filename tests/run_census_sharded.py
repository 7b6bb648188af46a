#!/usr/bin/env python3
"""torchrun worker: mdn_constraint_census on a session split over WORLD_SIZE ranks (mdn_session_set_shard world > 1) is
refused with MDN_ERR_UNSUPPORTED before any device work, and the session runs the census once the split is removed.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/run_census_sharded.py

tests/test_constraint_census.py runs it on the CPU kernel emulator (MDN_ALLOW_EMULATOR=1 MDN_EMU_SHM=1, gloo)."""
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
    import helpers as H
    import test_airs
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    wl, bld = test_airs.fib_product_workload([5])
    s = B.Session(params, local)
    s.set_shard(rank, world, pkg.parallel.make_allgather_callback(dev_name))
    try:
        s.constraint_census(wl.statement, wl.matrices, ch, aux_builder=B.AUX_BUILDER(bld))
        raise SystemExit("census on a split session was not refused")
    except B.ProverError as e:
        assert str(e).startswith("[-4]") and "split over ranks" in str(e), str(e)
    s.set_shard(0, 1, pkg.parallel.make_allgather_callback(dev_name))
    c, f, t, _ = s.constraint_census(wl.statement, wl.matrices, ch, aux_builder=B.AUX_BUILDER(bld))
    assert c.first.holds == 1 and c.violations == 0 and not f and not t
    s.close()
    dist.barrier()
    print(f"CENSUS_SHARD_REFUSED_OK rank={rank} world={world}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
