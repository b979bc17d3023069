"""Worker of tests/test_host_motion_segments_fake_runtime.py: Motions on in-process clusters of 64 and 65 segments over the no-op
runtime of tests/fake_runtime.py (LD_PRELOADed by the test; kernels are no-ops, "device" memory is zeroed host memory).  Prints
one "MOTIONSEGS {json}" line per case as soon as it returns.  Not a test by itself."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from cloudberry_b200 import capi  # noqa: E402
from cloudberry_b200 import plan as P  # noqa: E402


def run(cl, plan):
    """Cluster.run, with the code of the segment that failed (Cluster.run reports -1 and the segment's message)"""
    E = cl.E
    rc = E.cb_cluster_init_plan(cl.h, P.plan_ptr(plan))
    if rc:
        msg = E.cb_cluster_error(cl.h).decode()
        E.cb_cluster_end(cl.h)
        return {"code": rc, "msg": msg}
    rows, code, msg = 0, 0, ""
    try:
        while True:
            slot = E.cb_cluster_next(cl.h)
            err = E.cb_cluster_error(cl.h)
            if err:
                msg = err.decode()
                code = next((c for c in (E.cb_cluster_estate(cl.h, s).contents.es_errcode for s in range(cl.nsegs)) if c), -1)
                break
            if not slot or slot.contents.tts_empty:
                break
            rows += 1
    finally:
        E.cb_cluster_end(cl.h)
    return {"code": code, "msg": msg, "rows": rows}


def main():
    ctx = capi.Context(0)
    n = 1000
    rel = capi.DeviceRelation(ctx, n, [P.INT4, P.INT8], name="t")
    cols = [np.arange(n, dtype=np.int32), np.arange(n, dtype=np.int64)]     # alive until the asynchronous copies are done
    for c, a in enumerate(cols):
        ctx.check(ctx.L.cbgpu_rel_load_column(rel.h, c, a.ctypes.data, None))
    ctx.sync()
    scan = P.SeqScan(1, [("k", P.Var(1, 1, P.INT4)), ("v", P.Var(1, 2, P.INT8))])
    for nsegs in (64, 65):
        cl = capi.Cluster(ctx, [[rel]] * nsegs)
        for name, plan in (("hash", P.Motion(scan, P.MOTIONTYPE_HASH, [P.out_var(scan, 1)])),
                           ("hash_two_keys", P.Motion(scan, P.MOTIONTYPE_HASH, [P.out_var(scan, 2), P.out_var(scan, 1)])),
                           ("gather", P.Motion(scan, P.MOTIONTYPE_GATHER)),
                           ("broadcast", P.Motion(scan, P.MOTIONTYPE_BROADCAST))):
            before = ctx.launches()
            r = run(cl, plan)
            print("MOTIONSEGS " + json.dumps(dict(r, nsegs=nsegs, case=name, launches=ctx.launches() - before)), flush=True)
        cl.close()
    rel.free()
    ctx.close()


if __name__ == "__main__":
    main()
