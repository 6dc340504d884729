"""bench_configs.py -- BASELINE.json configs C2..C5 (python bench.py --config Cx [--gpus N] [--rows R]).

One JSON line per run: build Mvec/s (resident and e2e from pinned host memory), the per-kernel breakdown of one
profiled build, the assign kernel's roofline against the measured TENSOR peak (2*n*K*d flops), an IN-RUN ORACLE
CHECK of a row sample (partition ids + PQ codes bit-exact against oracle/ on the same model), a query batch with
recall against exact brute force, and a bounded CPU sample of the same per-row work.  Every rank of a --gpus N run
holds one shard of `rows` rows (weak scaling; --gpus 8 = the configuration at full size): the k-means loops
exchange packed partial sums once per iteration, everything else is local to the shard.
"""
import json
import os
import time

import numpy as np

NQ, TOPK = 10_000, 10


def _np_dtype(name):
    return {"f32": np.float32, "f16": np.float16, "bf16": np.uint16, "u8": np.uint8}[name]


def _to_f32(host, name):
    if name == "bf16":
        return (host.astype(np.uint32) << 16).view(np.float32)
    return host.astype(np.float32)


def make_data(torch, cfg, n, seed, device, queries=False):
    """Gaussian mixture with ncomp components in the configuration's element type (SURVEY 8d): f32 rows are unit
    normalised (ada-002 shape), f16 / bf16 are N(centre, 1), u8 are clipped integers (BigANN shape)."""
    d, ncomp, name = cfg["d"], cfg["ncomp"], cfg["dtype"]
    g = torch.Generator(device=device)
    g.manual_seed(4242)                                            # the mixture itself: same on every rank
    if name == "u8":
        centres = torch.randint(20, 236, (ncomp, d), device=device, generator=g, dtype=torch.int32).float()
        sigma = 12.0
    else:
        centres = torch.randn((ncomp, d), device=device, generator=g) * (3.0 if name != "f32" else 1.0)
        sigma = 1.0 if name != "f32" else 0.35
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "u8": torch.uint8}[name]
    out = torch.empty((n, d), dtype=tdt, device=device)
    g.manual_seed(seed)
    step = max(1, (1 << 27) // d)
    for s in range(0, n, step):
        e = min(n, s + step)
        comp = torch.randint(0, ncomp, (e - s,), device=device, generator=g)
        x = centres[comp] + torch.randn((e - s, d), device=device, generator=g) * sigma
        if name == "f32":
            x = x / x.norm(dim=1, keepdim=True)
        elif name == "u8":
            x = torch.clamp(torch.round(x), 0, 255)
        out[s:e] = x.to(tdt)
    return out


def run(args, cfg, B):
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    import torch
    import torch.distributed as dist

    import lance_b200 as lb
    from lance_b200 import _lib
    if lb.device_count() < 1:
        raise SystemExit("bench.py: no CUDA device (lance_b200 has no CPU fallback)")
    torch.cuda.set_device(local_rank)
    lb.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
        from tools import dist_util
        dist_util.init_comm(dist)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        lb.synchronize()

    def max_over_ranks(x):
        if world > 1:
            t = torch.tensor([x], dtype=torch.float64, device=device)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t.item())
        return x

    n = args.rows or cfg["rows"]
    d, K, M, name, metric, kind = cfg["d"], cfg["K"], cfg["M"], cfg["dtype"], cfg["metric"], cfg["kind"]
    npdt = _np_dtype(name)
    esize = np.dtype(npdt).itemsize
    t_gen = time.perf_counter()
    data_t = make_data(torch, cfg, n, 1000 + rank, device)
    queries_t = make_data(torch, cfg, NQ, 77, device)
    torch.cuda.synchronize()
    t_gen = time.perf_counter() - t_gen
    view = data_t.view(torch.uint16) if name == "bf16" else data_t
    qview = queries_t.view(torch.uint16) if name == "bf16" else queries_t
    data_dev, q_dev = B.wrap_tensor(lb, view, npdt), B.wrap_tensor(lb, qview, npdt)
    row_base = rank * n
    rid_t = torch.arange(row_base, row_base + n, dtype=torch.int64, device=device)
    rid_dev = B.wrap_tensor(lb, rid_t, np.uint64)

    def build(src=data_dev, rids=rid_dev):
        if kind == "flat":
            return lb.IvfFlatIndex.build(src, metric, num_partitions=K, seed=7, row_ids=rids, bf16=(name == "bf16"))
        return lb.IvfPqIndex.build(src, metric, lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, seed=7), row_ids=rids)

    for _ in range(args.warmup):
        build().close()
    sampler = B.ClockSampler(local_rank)
    sampler.start()
    time.sleep(0.3)
    barrier()
    lb.launch_count(reset=True)
    t_wall0 = time.time()
    lb.timer_start()
    stats = None
    for _ in range(args.steps):
        ix = build()
        stats = ix.stats
        ix.close()
    ms_step = max_over_ranks(lb.timer_stop() / args.steps)
    barrier()
    t_wall1 = time.time()
    launches = lb.launch_count()
    clocks = sampler.summary(t_wall0, t_wall1)
    value = world * n / (ms_step * 1e-3) / 1e6

    # ---- one profiled build: per-kernel CUDA-event times ---------------------------------------------------
    lb.profile.reset()
    lb.profile.enable(True)
    lb.timer_start()
    ix = build()
    ms_prof = lb.timer_stop()
    lb.profile.enable(False)
    fams = {f: {"launches_per_step": c, "ms_per_step": ms, "share": ms / ms_prof}
            for f, (c, ms) in sorted(lb.profile.dump().items(), key=lambda kv: -kv[1][1])}
    hbm_peak, tensor_peak, peak_src = B.peaks()
    filt = next((f for f in ("transform:tc_filter_general16", "transform:tc_filter_general", "transform:tc_filter") if f in fams), None)
    roofline = None
    if filt:
        flops = 2.0 * n * K * d
        ms = fams[filt]["ms_per_step"]
        nl = fams[filt]["launches_per_step"]
        ach = flops / (ms * 1e-3) / 1e12
        roofline = {"kernel": filt, "bound": "tensor", "achieved": ach, "peak": tensor_peak, "unit": "TFLOP/s",
                    "frac": ach / tensor_peak,
                    "peak_source": peak_src + "; " + ("the kernel runs f16 / bf16 wgmma on the native 16-bit rows"
                                                      if filt.endswith("16") else "the kernel runs tf32 wgmma on f32 rows (half the bf16 rate)"),
                    "algorithmic_flops_per_launch": flops / nl, "avg_launch_ms": ms / nl, "launches": nl,
                    "hbm_GBps_streaming_x": n * d * esize / (ms * 1e-3) / 1e9}
    top = dict(list(fams.items())[:14])

    # ---- in-run oracle check on a row sample ------------------------------------------------------------------
    from oracle import binding as ob
    threads = ob.nthreads_default()
    S = min(n, 4096)
    rng = np.random.default_rng(5 + rank)
    rows = np.sort(rng.choice(n, S, replace=False))
    sel = torch.from_numpy(rows).to(device)
    sample_raw = (data_t[sel].view(torch.int16).cpu().numpy().view(np.uint16) if name == "bf16" else view[sel].cpu().numpy())
    sample = _to_f32(sample_raw, name)
    parts = ix.export()
    cent = parts["centroids"]
    src = ob.normalize_rows(sample, nthreads=threads) if metric == "cosine" else sample
    t0 = time.perf_counter()
    p_ref, _, v_ref = ob.compute_membership(cent, src, metric="dot" if metric == "dot" else "l2", nthreads=threads)
    t_cpu_assign = time.perf_counter() - t0
    parity = {"rows_checked": int(S), "oracle_threads": threads}
    codes_ref = None
    t_cpu_encode = 0.0
    if kind == "pq":
        res = ob.compute_residual(cent, src, p_ref, nthreads=threads)
        t0 = time.perf_counter()
        codes_ref = ob.pq_encode(parts["codebook"], res, nthreads=threads)
        t_cpu_encode = time.perf_counter() - t0
        # (a) the device transform on the same sample with the same model
        p_dev, c_dev, v_dev = lb.ivfpq_transform(cent, parts["codebook"], sample, distance_type=metric)
        parity["transform_sample_part_ids_equal"] = bool(np.array_equal(p_dev, p_ref))
        parity["transform_sample_codes_equal"] = bool(np.array_equal(c_dev, codes_ref))
    else:
        p_dev, _, _ = lb.compute_partitions(cent, src)
        parity["sample_part_ids_equal"] = bool(np.array_equal(p_dev, p_ref))
    # (b) what the BUILD stored for those rows
    if n <= 30_000_000:
        pos = np.empty(n, np.int64)
        pos[(parts["row_ids"] - np.uint64(row_base)).astype(np.int64)] = np.arange(len(parts["row_ids"]))
        sizes = np.diff(parts["part_offsets"]).astype(np.int64)
        part_of_pos = np.repeat(np.arange(K, dtype=np.uint32), sizes)
        parity["index_part_ids_equal"] = bool(np.array_equal(part_of_pos[pos[rows]], p_ref))
        if kind == "pq":
            parity["index_codes_equal"] = bool(np.array_equal(parts["codes"][pos[rows]], codes_ref))
        else:
            stored = parts["vectors"][pos[rows]]     # kept in the column's element type
            parity["index_vectors_equal"] = bool(np.array_equal(stored, sample_raw if metric != "cosine" else src.astype(stored.dtype)))
        del pos, part_of_pos
    parity["ok"] = all(v for k, v in parity.items() if k.endswith("_equal"))

    # ---- query batch ------------------------------------------------------------------------------------------
    nprobes = cfg["nprobes"]
    ids_t = torch.empty((NQ, TOPK), dtype=torch.int64, device=device)
    d_t = torch.empty((NQ, TOPK), dtype=torch.float32, device=device)
    ids_dev, d_dev = B.wrap_tensor(lb, ids_t, np.uint64), B.wrap_tensor(lb, d_t, np.float32)
    fn = ix.search if world == 1 else ix.search_sharded
    for _ in range(2):
        fn(q_dev, TOPK, nprobes, out=(ids_dev, d_dev))
    barrier()
    lb.timer_start()
    qsteps = max(2, args.steps)
    for _ in range(qsteps):
        fn(q_dev, TOPK, nprobes, out=(ids_dev, d_dev))
    q_ms = max_over_ranks(lb.timer_stop() / qsteps)
    NG = 200
    gi, gd = B.ground_truth(torch, data_t, queries_t[:NG], TOPK, row_base=row_base, cosine=(metric == "cosine"),
                            return_dists=True)
    if world > 1:   # exact top-k over ALL shards: gather every rank's exact list, keep the k nearest
        li = [torch.empty_like(gi) for _ in range(world)]
        ld = [torch.empty_like(gd) for _ in range(world)]
        dist.all_gather(li, gi)
        dist.all_gather(ld, gd)
        ci, cd = torch.cat(li, 1), torch.cat(ld, 1)
        o = torch.topk(cd, TOPK, dim=1, largest=False).indices
        gi = torch.gather(ci, 1, o)
    gt_local = gi.cpu().numpy()
    got = ids_t[:NG].cpu().numpy()
    recall = float(np.mean([len(set(got[i].tolist()) & set(gt_local[i].tolist())) / TOPK for i in range(NG)]))
    query = {"qps": NQ / (q_ms * 1e-3), "ms_per_batch": q_ms, "batch": NQ, "k": TOPK, "nprobes": nprobes,
             "recall_at_10": recall, "indexed_rows": world * n,
             "note": "recall against exact brute force over ALL shards; sharded runs merge in the library (lb2_index_search_sharded)"}
    ix.close()

    # ---- e2e: pinned host -> build -> export to host ------------------------------------------------------------
    e2e = None
    try:
        pin = lb.PinnedArray((n, d), npdt)
        import ctypes as C
        _lib.check(lb.lib().lb2_memcpy(C.c_void_p(pin.ptr), C.c_void_p(data_t.data_ptr()), C.c_size_t(n * d * esize)))
        del data_dev, view, data_t, gt_local      # the device copy of the dataset makes room for the host-fed build
        torch.cuda.empty_cache()
        barrier()
        t0 = time.perf_counter()
        ixh = build(pin, None)
        ph = ixh.export()
        barrier()
        e2e_ms = max_over_ranks((time.perf_counter() - t0) * 1e3)
        d2h = int(sum(v.nbytes for v in ph.values()))
        ixh.close()
        e2e = {"value": world * n / (e2e_ms * 1e-3) / 1e6, "unit": "Mvec/s", "ms_per_step": e2e_ms, "steps": 1,
               "h2d_bytes_per_step": n * d * esize, "d2h_bytes_per_step": d2h}
        del ph
        pin.free()
    except Exception as ex:  # host memory for the pinned copy is the usual limit
        e2e = {"value": None, "unavailable": str(ex)[:200]}

    # ---- CPU sample: the oracle's per-row transform on the sample rows -------------------------------------------
    cpu_baseline = None
    if rank == 0 and not args.no_cpu_baseline:
        t = t_cpu_assign + t_cpu_encode
        cpu_baseline = {"value": S / t / 1e6, "unit": "Mvec/s", "cores": threads, "kind": "port",
                        "sample": f"partition id + residual + PQ code of {S} rows with the trained model (training is not "
                                  f"timed on the CPU: favours the CPU arm); {t:.2f} s",
                        "assign_s": t_cpu_assign, "encode_s": t_cpu_encode}
    sampler.stop()
    if rank == 0:
        line = {
            "metric": "ivf_flat_index_build_mvec_per_s" if kind == "flat" else "ivf_pq_index_build_mvec_per_s",
            "value": value, "unit": "Mvec/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": name,
            "data": "synthetic",
            "config": {"workload": cfg["desc"], "rows_per_gpu": n, "rows_total": world * n, "config_rows_total": cfg["total"],
                       "d": d, "num_partitions": K, "num_sub_vectors": M, "metric": metric,
                       "cache": f"inputs ({n * d * esize / 1e9:.1f} GB per GPU) larger than L2 (50 MB)", "k": TOPK, "nprobes": nprobes,
                       "data_generation_s": t_gen},
            "clocks": clocks, "e2e": e2e, "gpu_launches": launches,
            "build_phases_ms": {"ivf_train": stats.ms_ivf_train, "pq_train": stats.ms_pq_train, "transform": stats.ms_transform,
                                "group": stats.ms_group, "ivf_iters": stats.ivf_iters, "pq_iters_max": stats.pq_iters_max},
            "kernels_top": top, "roofline": roofline, "parity": parity, "query": query, "cpu_baseline": cpu_baseline,
        }
        print(json.dumps(line))
    if world > 1:
        from lance_b200 import parallel
        parallel.comm_destroy()
        dist.destroy_process_group()
