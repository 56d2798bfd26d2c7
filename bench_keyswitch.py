#!/usr/bin/env python
"""bench_keyswitch.py -- key-switch (reLinearize + mod-down) throughput, BASELINE configs 3 and 4.

  --mode sharded  : ONE stream of ciphertexts, every ciphertext's rows sharded by RNS prime index over the
                    N GPUs (helib_b200/sharded.py; all-gather of the digit y-rows and of the special-prime
                    y-rows over NCCL/NVLink).  scaling = "strong".  BASELINE config 4 (CKKS N=2^16, 29+15 primes).
  --mode replicas : independent ciphertexts per GPU, evk replicated, no collective.  scaling = "weak".
                    BASELINE config 3 (BGV m=2^17 p=257 bits=1500 c=3) by default.

  --prg           : instead, the device expansion of key-switching rows from a PRG seed (hb_poly_randomize):
                    all a_i of a config-3 matrix (3 x 35 rows, N = 2^16) and of config 2's, ms per matrix over
                    repeated runs, GB/s of key stream consumed, the count and fill passes separately.
  --seeded        : instead, key-switching matrices held as b_i plus their PRG seed (hb_poly_create_seeded: every key
                    switch regenerates the a_i rows it reads) against the same matrices expanded, alternated in one
                    process: config-3 relinearise + mod-down in groups of 64, config-2 multiply + relinearise + mod-down
                    at batch 32, and hoisted rotations on config 5's ring (m = 21845) at batch 8 with one matrix per
                    amount.  Both rates, an in-run bit-identity check, device bytes per matrix and creation time.

Launch: python bench_keyswitch.py [--mode ...]            (1 GPU)
        python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench_keyswitch.py --gpus N ...
Prints one JSON line on rank 0 (key-switches/s = 3-part -> 2-part over S|special, then mod-down to S).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {
    "cfg4": {"name": "ckks_m2^17_bits1700_c2 (l=29,K=15,d=2)", "m": 1 << 17, "p": -1, "r": 1, "bits": 1700, "c": 2},
    "cfg3": {"name": "bgv_m2^17_p257_bits1500_c3 (l=26,K=9,d=3)", "m": 1 << 17, "p": 257, "r": 1, "bits": 1500, "c": 3},
}
ROW = (1 << 16) * 8
PRG_WORKLOADS = {
    "cfg3": {"name": "bgv_m2^17_p257_bits1500_c3", "m": 1 << 17, "p": 257, "r": 1, "bits": 1500, "c": 3},
    "cfg2": {"name": "ckks_m2^17_bits1190_c2", "m": 1 << 17, "p": -1, "r": 1, "bits": 1190, "c": 2},
}
PRG_SEED = 0xB7E151628AED2A6ABF7158809CF4F3C762E7160F38B4DA56A784D9045190CFEF


def bench_prg(args):
    """ms per key-switching matrix expanded from its seed: SetSeed(prgSeed); a[i].randomize() for every digit i over
    ctxt|special, one hb_poly_randomize call.  The rows are checked against the vectorised oracle, which also gives the
    exact number of 2048-byte key-stream buffers the matrix consumes."""
    import numpy as np
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ntl_prg_np as npg
    from bench import gpu_identity
    from helib_b200 import Chain, Engine
    out = {"metric": "prg_matrix_expansion", "unit": "ms/matrix", "gpu": gpu_identity(0), "steps": args.steps, "reps": args.reps, "workloads": []}
    for key, wl in PRG_WORKLOADS.items():
        ch = Chain(wl["m"], wl["p"], wl["r"], wl["bits"], wl["c"])
        E = Engine(wl["m"], ch.primes, None, ch.digits, ch.special)
        full = ch.ctxt + ch.special
        n = len(ch.digits)
        A = [E.poly() for _ in range(n)]
        E.randomize(A, full, PRG_SEED)
        bs = npg.BufferStream(PRG_SEED)
        for d in range(n):
            ref = npg.randomize_rows(ch.primes, E.N, full, bs)
            got = A[d].download(full)
            assert all(np.array_equal(got[i], ref[i]) for i in full), f"{key}: device rows differ from the oracle"
        stream_bytes = bs.next * 2048
        for _ in range(max(1, args.warmup)):
            E.randomize(A, full, PRG_SEED)
        runs = []
        for _ in range(args.reps):
            E.mark_begin()
            for _ in range(args.steps):
                E.randomize(A, full, PRG_SEED)
            runs.append(E.mark_end() / args.steps)
        E.profile(True)
        E.randomize(A, full, PRG_SEED)
        E.profile(False)
        prof = {r["kernel"]: {"launches": r["launches"], "ms": round(r["ms"], 4)} for r in E.profile_results()}
        med = float(np.median(runs))
        out["workloads"].append({
            "workload": wl["name"], "N": E.N, "polys": n, "rows_per_poly": len(full),
            "key_stream_MB": round(stream_bytes / 1e6, 2),
            "ms_per_matrix": {"median": round(med, 4), "min": round(min(runs), 4), "max": round(max(runs), 4)},
            "key_stream_GBps": round(stream_bytes / (med / 1e3) / 1e9, 1),
            "passes": prof,
        })
        E.close()
    print(json.dumps(out))


SEEDED_WORKLOADS = {
    "cfg3_relin_moddown": {"name": "bgv_m2^17_p257_bits1500_c3 relinearize+scale_down", "m": 1 << 17, "p": 257, "bits": 1500, "c": 3, "batch": 64},
    "cfg2_mul_relin_moddown": {"name": "ckks_m2^17_bits1190_c2 mul_relin_moddown", "m": 1 << 17, "p": -1, "bits": 1190, "c": 2, "batch": 32},
    "cfg5_hoisted_rotation": {"name": "bgv_m21845_p2_bits580_c2_bootstrappable automorph_keyswitch_digits", "m": 21845, "p": 2, "bits": 580, "c": 2,
                              "batch": 8, "bootstrappable": True, "amounts": 4},
}


def _seeded_workload(args, key, wl, ch, E):
    import time
    import numpy as np
    N, npr, B = E.N, E.np, wl["batch"]
    p = 1 if ch.p == -1 else ch.p
    S = ch.ctxt
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    rng = np.random.Generator(np.random.Philox(20261015))

    def rand(idx):
        x = np.zeros((npr, N), dtype=np.uint64)
        for i in idx:
            x[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
        return x

    nkeys = wl.get("amounts", 1)
    seeds = [PRG_SEED + j for j in range(nkeys)]
    b0 = E.stats()["device_bytes"]
    EA = [[E.poly() for _ in range(nd)] for _ in range(nkeys)]
    expanded_bytes = (E.stats()["device_bytes"] - b0) // nkeys
    for A, sd in zip(EA, seeds):
        E.randomize(A, full, sd)
    E.sync()
    b1 = E.stats()["device_bytes"]
    SA = [E.seeded(nd, full, sd) for sd in seeds]
    seeded_bytes = (E.stats()["device_bytes"] - b1) // nkeys
    create_ms = []
    for _ in range(5):
        E.sync()
        t0 = time.perf_counter()
        tmp = E.seeded(nd, full, PRG_SEED)
        E.sync()
        create_ms.append((time.perf_counter() - t0) * 1e3)
        del tmp
    EB = [[E.poly(rand(full), full) for _ in range(nd)] for _ in range(nkeys)]

    if key == "cfg3_relin_moddown":
        Sp = full
        src = [[rand(S) for _ in range(3)] for _ in range(B)]
        C = [[E.poly(x[k], S) for k in range(3)] for x in src]
        C0, C1, C2 = ([c[k] for c in C] for k in range(3))

        def load():
            for c, x in zip(C, src):
                for k in range(3):
                    c[k].upload(x[k], S)

        def step(A, j=0):
            E.relinearize(C0, C1, C2, S, A[0], EB[0])
            E.scale_down(C0 + C1, Sp, S, p)
        outputs, out_idx = (lambda: C0 + C1), S
    elif key == "cfg2_mul_relin_moddown":
        S_in, S = ch.ctxt, ch.ctxt[:-1]
        src = [[rand(S_in) for _ in range(4)] for _ in range(B)]
        P = [[E.poly(x[k], S_in) for k in range(4)] for x in src]
        A0, A1, B0, B1 = ([q[k] for q in P] for k in range(4))

        def load():
            for q, x in zip(P, src):
                for k in range(4):
                    q[k].upload(x[k], S_in)

        def step(A, j=0):
            E.mul_relin_moddown(A0, A1, B0, B1, S_in, S, p, A[0], EB[0])
        outputs, out_idx = (lambda: A0 + A1), S
    else:
        Sp = full
        C0 = [E.poly(rand(S), S) for _ in range(B)]
        digs = E.break_into_digits([E.poly(rand(S), S) for _ in range(B)], S)
        O0, O1 = [E.poly() for _ in range(B)], [E.poly() for _ in range(B)]
        amounts = [t for t in range(2, wl["m"]) if np.gcd(t, wl["m"]) == 1][:nkeys]

        def load():
            pass

        def step(A, j=None):
            for a in (range(nkeys) if j is None else [j]):
                E.automorph_keyswitch_digits(digs, S, C0, amounts[a], A[a], EB[a], O0, O1)
        outputs, out_idx = (lambda: O0 + O1), Sp

    # in-run check: the same inputs through both forms give the same output rows
    got = []
    for A in (EA, SA):
        load()
        step(A, 0) if key == "cfg5_hoisted_rotation" else step(A)
        got.append([x.download(out_idx)[out_idx] for x in outputs()])
    identical = all(np.array_equal(a, b) for a, b in zip(*got))
    per_call = nkeys if key == "cfg5_hoisted_rotation" else 1
    runs = {"expanded": [], "seeded": []}
    for form, A in (("expanded", EA), ("seeded", SA)):
        for _ in range(max(1, args.warmup)):
            step(A)
    for _ in range(args.reps):
        for form, A in (("expanded", EA), ("seeded", SA)):
            E.sync()
            E.mark_begin()
            for _ in range(args.steps):
                step(A)
            ms = E.mark_end() / (args.steps * per_call)
            runs[form].append(B / (ms / 1e3))
    med = {f: float(np.median(v)) for f, v in runs.items()}
    return {
        "workload": wl["name"], "N": N, "batch": B, "digits": nd, "rows_per_a": len(full), "matrices": nkeys,
        "rate_items_per_s": {f: {"median": round(med[f], 1), "min": round(min(v), 1), "max": round(max(v), 1)} for f, v in runs.items()},
        "seeded_vs_expanded": round(med["seeded"] / med["expanded"] - 1.0, 4),
        "outputs_bit_identical": identical,
        "device_bytes_per_matrix_a": {"expanded": expanded_bytes, "seeded": seeded_bytes},
        "device_bytes_per_matrix_a_and_b": {"expanded": 2 * expanded_bytes, "seeded": expanded_bytes + seeded_bytes},
        "create_seeded_ms": {"median": round(float(np.median(create_ms)), 3), "min": round(min(create_ms), 3)},
    }


def bench_seeded(args):
    """Expanded against seeded a_i in the key-switching entry points, alternated run by run in one process."""
    from bench import gpu_identity
    from helib_b200 import Chain, Engine
    out = {"metric": "seeded_keyswitch_matrices", "unit": "items/s", "gpu": gpu_identity(0), "steps": args.steps, "reps": args.reps,
           "workloads": []}
    for key, wl in SEEDED_WORKLOADS.items():
        ch = Chain(wl["m"], wl["p"], 1, wl["bits"], wl["c"], bootstrappable=wl.get("bootstrappable", False))
        E = Engine(wl["m"], ch.primes, None, ch.digits, ch.special)
        out["workloads"].append(_seeded_workload(args, key, wl, ch, E))   # its polys are freed on return
        E.close()
    print(json.dumps(out))
    if not all(w["outputs_bit_identical"] for w in out["workloads"]):
        sys.exit(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--mode", default="sharded", choices=["sharded", "replicas"])
    ap.add_argument("--workload", default=None)
    ap.add_argument("--no-graph", action="store_true", help="do not capture the step into a CUDA graph")
    ap.add_argument("--exchange", default="p2p", choices=["p2p", "gather"], help="sharded mode: peer stores from the producing kernel, or pack/all_gather/unpack")
    ap.add_argument("--profile", action="store_true", help="add a per-kernel table (CUDA events per launch, one eager step)")
    ap.add_argument("--prg", action="store_true", help="time the device expansion of key-switching rows from a PRG seed instead")
    ap.add_argument("--reps", type=int, default=5, help="--prg: timed runs of --steps expansions each; --seeded: runs of each form")
    ap.add_argument("--seeded", action="store_true", help="time key switches with seeded against expanded a_i instead")
    args = ap.parse_args()
    if args.prg:
        return bench_prg(args)
    if args.seeded:
        return bench_seeded(args)
    import numpy as np
    import torch
    import torch.distributed as dist
    from helib_b200 import Chain, Engine
    from helib_b200.sharded import ShardedKeySwitch

    wl = WORKLOADS[args.workload or ("cfg4" if args.mode == "sharded" else "cfg3")]
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ch = Chain(wl["m"], wl["p"], wl["r"], wl["bits"], wl["c"])
    E = Engine(wl["m"], ch.primes, None, ch.digits, ch.special, device=local)
    side = torch.cuda.Stream()            # the engine, torch index ops and NCCL all run ordered on this stream
    torch.cuda.set_stream(side)
    E.set_stream(side.cuda_stream)
    p = 1 if ch.p == -1 else ch.p ** ch.r
    N, npr, B = E.N, E.np, args.batch
    S = ch.ctxt
    full = ch.ctxt + ch.special
    nd = len(ch.digits)
    sharded = args.mode == "sharded"
    KS = ShardedKeySwitch(E, ch.ctxt, ch.special, ch.digits, rank=rank if sharded else 0, world=world if sharded else 1, device=f"cuda:{local}", p2p=(args.exchange == "p2p"))
    rng = np.random.Generator(np.random.Philox(20260922 + (4 if sharded else 3) + (0 if sharded else 1000 * rank)))

    def rand_rows(idx):
        out = np.zeros((npr, N), dtype=np.uint64)
        for i in idx:
            out[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
        return out

    own_full, oS = KS.owned(full), KS.owned(S)
    EA = [E.poly(rand_rows(own_full), own_full) for _ in range(nd)]
    EB = [E.poly(rand_rows(own_full), own_full) for _ in range(nd)]
    C = [[E.poly(rand_rows(oS), oS) for _ in range(3)] for _ in range(B)]
    digs = [[E.poly() for _ in range(nd)] for _ in range(B)]
    C0, C1, C2 = ([c[k] for c in C] for k in range(3))

    def step():
        Sp = KS.relinearize(C0, C1, C2, S, EA, EB, digs)
        KS.mod_down(C0 + C1, Sp, S, p)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(max(3, args.warmup)):
        step()
    E.reset_stats()
    step()
    launches_per_step = E.stats()["launches"]
    barrier()
    # The sharded step is ~100 small launches + 3 collectives: capture it once into a CUDA graph
    # (engine kernels and torch's NCCL all-gathers are all ordered on torch's current stream).
    graphed = False
    run = step
    if not args.no_graph:
        try:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                step()
            run = g.replay
            graphed = True
            for _ in range(2):
                run()
        except Exception as ex:   # fall back to eager launches
            if rank == 0:
                print(f"[bench_keyswitch] CUDA graph capture failed ({type(ex).__name__}: {ex}); running eagerly", file=sys.stderr)
            run = step
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        run()
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    launches = launches_per_step * args.steps
    if world > 1:
        t = torch.tensor([ms], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    kernels = None
    if args.profile:
        E.profile(True)
        step()
        E.profile(False)
        prof = sorted(E.profile_results(), key=lambda r: -r["ms"])
        kernels = [{"kernel": r["kernel"], "launches": r["launches"], "ms": round(r["ms"], 4)} for r in prof]
        kernels.append({"kernel": "sum_of_engine_kernels", "launches": sum(r["launches"] for r in prof), "ms": round(sum(r["ms"] for r in prof), 4)})
    total = (B if sharded else B * world) * args.steps
    if rank == 0:
        l, K, d = len(S), len(ch.special), nd
        bks = ROW * (3 * l + 2 * d * (l + K) + 2 * l)      # SURVEY 8d: B_ks = 8N*[3l + 2d(l+K) + 2l]
        from bench import peaks
        peak, peak_kind = peaks()
        v = total / (ms / 1000.0)
        print(json.dumps({
            "metric": "key_switches_per_s", "value": v, "unit": "keyswitch/s", "n_gpus": world, "steps": args.steps, "warmup": max(3, args.warmup),
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "strong" if sharded else "weak", "vs_baseline": None,
            "dtype": "u64 (RNS limbs < 2^60)", "data": "synthetic",
            "config": {"workload": wl["name"], "mode": args.mode, "exchange": (args.exchange if (sharded and world > 1) else None), "N": N, "l": l, "K": K, "digits": d, "batch": B, "ptxt_space": p,
                       "collectives_per_keyswitch": (d + 1) if (sharded and world > 1) else 0,
                       "all_gather_bytes_per_keyswitch": (l + 2 * K) * ROW if (sharded and world > 1) else 0, "alg_bytes_per_keyswitch": bks},
            "alg_roofline": {"achieved_GBps": v * bks / 1e9, "peak_GBps": peak * world, "frac": v * bks / 1e9 / (peak * world), "peak_kind": peak_kind},
            "gpu_launches": launches, "cuda_graph": graphed, "kernels": kernels,
        }))
    # Leave without tearing NCCL down: destroy_process_group() after a captured graph that contains
    # collectives can block for minutes; the results are already printed.
    sys.stdout.flush()
    sys.stderr.flush()
    if world > 1:
        torch.cuda.synchronize()
        os._exit(0)


if __name__ == "__main__":
    main()
