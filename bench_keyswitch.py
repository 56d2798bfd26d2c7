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
    ap.add_argument("--reps", type=int, default=5, help="--prg: timed runs of --steps expansions each")
    args = ap.parse_args()
    if args.prg:
        return bench_prg(args)
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
