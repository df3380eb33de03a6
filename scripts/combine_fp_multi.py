"""The float8 overflow rule of the Finalize step across datanodes (gx_result_combine), on N GPUs:
two finite partial sums whose merge leaves the float8 range are GX_ERR_OVERFLOW on the datanode that owns the
group; an infinite partial (an infinite input) merged with a finite one is Infinity, not an error.  Both
combine paths: the all-gather of small results and the redistribute of records (GX_NO_GATHER_COMBINE=1).
Launch with torchrun:

    torchrun --nproc-per-node 2 scripts/combine_fp_multi.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import opentenbase_b200 as g  # noqa: E402


def one_case(ctx, rank, x0):
    """group 7 holds x0 on rank 0; elsewhere x0 again when it is finite (1e308 per datanode), else 1.0"""
    x7 = x0 if rank == 0 or np.isfinite(x0) else 1.0
    t = ctx.table_from([g.GX_INT4, g.GX_FLOAT8], [np.array([7, 9], np.int32), np.array([x7, 2.5])])
    plan = g.make_plan(group_cols=[(0, 0)], aggs=[(g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)]), (g.GX_AGG_COUNT_STAR, [])], est_groups=4)
    res = ctx.hash_agg(t, plan)
    try:
        res.combine()
        keys, aggs, _ = res.fetch()
        out = ("ok", {int(k): float(v) for k, v in zip(keys[:, 0], aggs[:, 0])})
    except g.GxError as e:
        out = ("error", e.status)
    res.free(); t.free()
    return out


def main():
    import torch
    import torch.distributed as dist
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = g.Context(local)
    box = [g.Context.unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    ctx.comm_init(rank, world, box[0])
    ctx.set_shardmap(world)
    ok = True
    for case, x0 in (("finite", 1e308), ("inf", np.inf)):
        got = one_case(ctx, rank, x0)
        allgot = [None] * world
        dist.all_gather_object(allgot, got)
        if rank == 0:
            errors = [s for k, s in allgot if k == "error"]
            groups = {}
            for k, v in allgot:
                if k == "ok":
                    groups.update(v)
            if case == "finite":
                good = bool(errors) and all(s == g.GX_ERR_OVERFLOW for s in errors) and groups.get(9, 2.5 * world) == 2.5 * world
            else:
                good = not errors and groups.get(7) == np.inf and groups.get(9) == 2.5 * world
            print(f"{os.environ.get('GX_NO_GATHER_COMBINE', '0')} {case}: {allgot} -> {'pass' if good else 'FAIL'}", flush=True)
            ok = ok and good
    if rank == 0 and ok:
        print("OK combine overflow rule", flush=True)
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
