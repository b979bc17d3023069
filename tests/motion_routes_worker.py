"""Worker of tests/test_gpu_motion_routes.py::test_direct_motion_routes: run under torch.distributed.run, one process per segment,
every rank on one device, the interconnect the peer-memory windows (CB_BOOT=gloo).  The PARTITION sink stores each row straight
into its destination's window from inside the kernel.  Every rank builds all shards from one seed, runs the oracle over all of
them, runs its own shard through the executor and checks that the rows delivered to it are the oracle's rows for its segment.
Rank 0 prints MOTION ROUTES PASS when every rank agreed.  Not a test by itself."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import numpy as np
    import torch
    import torch.distributed as dist
    from cloudberry_b200 import capi
    from oracle import oracle as O
    from gpu_util import to_device
    from test_gpu_motion_routes import placement, scan_motion, split, table

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    ctx = capi.Context(0)

    def allgather(mine):
        box = [None] * world
        dist.all_gather_object(box, mine)
        return box
    motion = capi.Motion(ctx, rank, world, allgather=allgather)
    ok = motion.direct()
    if not ok:
        print("MOTION ROUTES FAIL: rank %d: no peer-memory path" % rank)
    n = 20011
    cases = [(k, "even", None) for k in ("int4", "int8_alias", "int8_fold", "date", "float8", "bpchar1", "bool", "dict8", "dict32",
                                         "mixed4", "null_one", "null_all")]
    cases += [("int4", "even", "payload_nulls"), ("mixed2", "hole", None)]
    for keyname, how, extra in cases:
        nl = (np.random.default_rng(5).random(n) < 0.3).astype(np.uint8) if extra else None
        pair = table(n, keyname, seed=17, payload_nulls=nl)
        segs_o, segs_p = split(pair, world, how)
        plan = scan_motion(pair[0])
        want = O.execute(plan, segs_o)
        wp = placement([0] * sum(1 for s in want.segments if s == rank), [r for s, r in zip(want.segments, want.rows) if s == rank])
        for generic in (False, True):
            dev = to_device(ctx, segs_p[rank])
            ex = capi.Executor(ctx, dev, force_generic=generic, motion=motion)
            try:
                got = ex.run(plan)
            finally:
                ex.close()
                for d in dev:
                    d.free()
            gp = placement(got.segments, got.rows)
            if gp != wp:
                ok = False
                print("MOTION ROUTES FAIL: rank %d, keys %s, %s senders, %s, generic %s: %d rows missing, %d extra"
                      % (rank, keyname, how, extra, generic, sum((wp - gp).values()), sum((gp - wp).values())))
    flag = torch.tensor([0 if ok else 1])
    dist.all_reduce(flag)
    if rank == 0 and flag.item() == 0:
        print("MOTION ROUTES PASS world", world, "cases", 2 * len(cases))
    motion.close()
    ctx.close()
    dist.destroy_process_group()
    sys.exit(1 if flag.item() else 0)


if __name__ == "__main__":
    main()
