"""Where the time of one multifrontal numeric factorisation goes, launch by launch, on the bench's headline workload (config C5, pose
graph of 2 500 SE3 poses, batch 2048, one linearization, damping 1e-3).

thb_front_factor_f64 / thb_front_factor_forward_f64 take a launch list and a count; here they are called with ONE row of the list at a
time, deepest first, on one chunk of the batch, with CUDA events around every call (--reps passes after two warm-up passes).  The arena
keeps the children's update matrices between the calls, so every call sees the inputs it has in the unsplit call.  (Each call clears
`info`; the workload is positive definite.)  Per launch the line holds what the plan says -- depth, class, threads per CTA, fronts,
dynamic shared memory, CTAs per SM, flops, bytes of panel, bytes of update matrix written and read, all per item -- and the measured ms
without and with the fused forward substitution; then totals per thread count and for the dense-path fronts, the Gram kernel alone
(whole batch), and the sum of the split calls against the unsplit call of the same chunk.  The GPU's name and power limit are printed
with the numbers.  Needs a CUDA device.

    python tools/front_launch_times.py [--batch 2048] [--reps 5] [--table] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

SM_COUNT, SMEM_PER_SM, SMEM_PER_CTA_RESERVED, THREADS_PER_SM = 132, 228 * 1024, 1024, 1024   # H100; 64 registers per thread


def small_threads(cls, smem):
    """Threads per CTA of a shared-memory launch (front_factor in thb_front.cu, default knobs)."""
    return 64 if cls == 0 else 128 if cls == 1 else 256 if smem <= 56 * 1024 else 512 if smem <= 113 * 1024 else 1024


def plan_columns(plan):
    """One dict per row of plan.launches with the columns that follow from the plan alone (flops and bytes per item)."""
    from theseus_b200.frontal import _front_cost
    A = plan.arrays
    w, b, sched, cp, cl = A["f_w"], A["f_b"], A["sched"], A["child_ptr"], A["child_list"]
    tri = lambda t: int(b[t]) * (int(b[t]) + 1) // 2 * 8   # the lower triangle of an update matrix
    rows = []
    for L in plan.launches:
        depth, cls, s0, cnt, smem = (int(v) for v in L[:5])
        ts = [int(t) for t in sched[s0:s0 + cnt]]
        row = dict(depth=depth, cls=cls, fronts=cnt, smem=smem if cls < 3 else None,
                   threads=small_threads(cls, smem) if cls < 3 else None,
                   r_max=max(int(w[t] + b[t]) for t in ts), w_max=max(int(w[t]) for t in ts),
                   mflop=sum(_front_cost(float(w[t]), float(b[t])) for t in ts) / 1e6,
                   panel_bytes=sum((int(w[t]) + int(b[t])) * int(w[t]) for t in ts) * 8,
                   update_written_bytes=sum(tri(t) for t in ts),
                   update_read_bytes=sum(tri(int(c)) for t in ts for c in cl[cp[t]:cp[t + 1]]))
        row["ctas_per_sm"] = (min(THREADS_PER_SM // row["threads"], SMEM_PER_SM // (smem + SMEM_PER_CTA_RESERVED), 32) if cls < 3 else None)
        rows.append(row)
    return rows


def class_totals(rows, keys):
    """Sums of `keys` (and launches, fronts) per thread count; the dense-path fronts under 'dense'."""
    out = {}
    for r in rows:
        t = out.setdefault(str(r["threads"]) if r["threads"] else "dense", dict(launches=0, fronts=0, **{k: 0.0 for k in keys}))
        t["launches"] += 1
        t["fronts"] += r["fronts"]
        for k in keys:
            t[k] += r[k]
    return out


def table(rows, totals):
    lines = ["depth cls thr fronts   smem cta/sm r_max w_max    MFLOP  panelKB  updWrKB  updRdKB  factor_ms  fused_ms"]
    for r in rows:
        lines.append("%5d %3d %4s %5d %7s %5s %5d %5d %8.2f %8.1f %8.1f %8.1f %9.3f %9.3f" % (
            r["depth"], r["cls"], r["threads"] or "-", r["fronts"], r["smem"] if r["smem"] is not None else "-", r["ctas_per_sm"] or "-",
            r["r_max"], r["w_max"], r["mflop"], r["panel_bytes"] / 1024, r["update_written_bytes"] / 1024, r["update_read_bytes"] / 1024,
            r["factor_ms"], r["factor_forward_ms"]))
    lines.append("threads launches fronts    MFLOP  factor_ms  fused_ms")
    for k, t in totals.items():
        lines.append("%7s %8d %6d %8.1f %9.2f %9.2f" % (k, t["launches"], t["fronts"], t["mflop"], t["factor_ms"], t["factor_forward_ms"]))
    return "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--table", action="store_true", help="also print the per-launch and per-class table")
    ap.add_argument("--json", help="also write the result line to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "front_launch_times.py needs a CUDA device"
    import theseus_b200 as th
    from theseus_b200 import _lib
    from theseus_b200.datasets import build_pose_graph_objective, pose_graph_sphere
    from theseus_b200.optimizer import convert_to_alpha_beta_damping_tensors
    from bench import C5_PER_RING, C5_RINGS
    from front_solve_phases import gpu_description

    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    B = args.batch
    data = pose_graph_sphere(C5_RINGS, C5_PER_RING, B, seed=1000, device=device)
    objective, _ = build_pose_graph_objective(th, data, device)
    opt = th.LevenbergMarquardt(objective, linear_solver_cls=th.BaspachoSparseSolver, linearization_cls=th.SparseLinearization,
                                max_iterations=1, linear_solver_kwargs=dict(layout="front"))
    solver, lin = opt.linear_solver, opt.linear_solver.linearization
    with torch.no_grad():
        lin.linearize()
    A64, b64 = lin.A_val.detach().double().contiguous(), lin.b.detach().double().contiguous()
    lam = torch.full((B,), 1e-3, dtype=torch.float64, device=device)
    alpha, beta = convert_to_alpha_beta_damping_tensors(lam, 1e-8, True, B, device, torch.float64)
    lib = _lib.load()
    Atb = solver._numeric_front(A64, b64, alpha, beta, forward=True)   # allocates the buffers, leaves the compact AtA and A^T b in them
    d, plan = solver._dev, solver._plan
    bufs, L = d["bufs"], d["launches"]
    nb, s = bufs["chunk"], _lib.stream_ptr()
    cols = L.shape[1]
    head = (_lib.ptr(bufs["factor"]), _lib.ptr(bufs["ata"]), solver._ata_size, _lib.ptr(alpha), _lib.ptr(beta), _lib.ptr(bufs["arena"]),
            _lib.ptr(bufs["ws"]) if d["max_np"] else None, bufs["ws"].numel(), _lib.ptr(bufs["info"]))
    fwd = (_lib.ptr(Atb), _lib.ptr(bufs["work"]), _lib.ptr(bufs["varena"]))

    def call(first, count, forward):
        rows = L.ctypes.data + first * cols * 8
        if forward:
            _lib.check(lib.thb_front_factor_forward_f64(C.byref(d["front"]), rows, count, *head, *fwd, nb, s), "front_factor_forward")
        else:
            _lib.check(lib.thb_front_factor_f64(C.byref(d["front"]), rows, count, *head, nb, s), "front_factor")

    def timed(calls):
        """ms per pass of each of `calls`, run one after the other per pass."""
        ev = [[(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in calls] for _ in range(args.reps)]
        for rep in range(-2, args.reps):
            for k, fn in enumerate(calls):
                if rep >= 0:
                    ev[rep][k][0].record()
                fn()
                if rep >= 0:
                    ev[rep][k][1].record()
        torch.cuda.synchronize()
        return [sum(ev[rep][k][0].elapsed_time(ev[rep][k][1]) for rep in range(args.reps)) / args.reps for k in range(len(calls))]

    def gram():
        nnz, m = A64.shape[1], b64.shape[1]
        _lib.check(lib.thb_gram_f64(C.byref(d["gram"]), B, _lib.ptr(A64), nnz, _lib.ptr(b64), m, _lib.ptr(bufs["ata"]), solver._ata_size,
                                    _lib.ptr(Atb), _lib.ptr(bufs["AtA_diag"]), s), "gram(front)")

    rows = plan_columns(plan)
    n = L.shape[0]
    whole = {}
    for key, forward in (("factor_ms", False), ("factor_forward_ms", True)):
        for r, ms in zip(rows, timed([lambda q=q, f=forward: call(q, 1, f) for q in range(n)])):
            r[key] = ms
        whole[key] = timed([lambda f=forward: call(0, n, f)])[0]
    gram_ms = timed([gram])[0]
    keys = ("mflop", "panel_bytes", "update_written_bytes", "update_read_bytes", "factor_ms", "factor_forward_ms")
    totals = class_totals(rows, keys)
    split = {k: sum(r[k] for r in rows) for k in whole}
    name, plim = gpu_description()
    line = dict(gpu=name, power_limit=plim, batch=B, chunk=nb, reps=args.reps, launches=rows, classes=totals, gram_ms_whole_batch=gram_ms,
                chunk_unsplit_ms=whole, chunk_split_sum_ms=split, split_minus_unsplit_ms={k: split[k] - whole[k] for k in whole})
    print(json.dumps(line))
    if args.table:
        print(table(rows, totals))
        print("Gram (batch %d) %.2f ms; one chunk of %d: unsplit %.2f / %.2f ms, sum of the split calls %.2f / %.2f ms (factor / fused); %s, %s" % (
            B, gram_ms, nb, whole["factor_ms"], whole["factor_forward_ms"], split["factor_ms"], split["factor_forward_ms"], name, plim))
    if args.json:
        with open(args.json, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
