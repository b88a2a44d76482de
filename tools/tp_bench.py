"""Micro-benchmark of the fused TP kernels vs the NCCL + GEMM baseline on the Llama-2-7B shapes.

torchrun --nproc-per-node N tools/tp_bench.py        → gpurun_out/tp_bench_tpN.json
Reports per op: fused µs, baseline µs (NCCL collective + own GEMM, and + cuBLAS), and the roofline
max(FLOPs / measured-GEMM-peak, NVLink-bytes / 770 GB/s) with the achieved fraction."""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timeit(fn, iters=20, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize(); dist.barrier()
    times = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e) * 1e3)
    times.sort()
    t = torch.tensor([times[len(times) // 2]], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    from neuronx_distributed_b200 import ops
    from neuronx_distributed_b200.ops import _fused_impl, gemm
    from neuronx_distributed_b200.parallel_layers import comm
    from neuronx_distributed_b200.parallel_layers import parallel_state as ps

    ps.initialize_model_parallel(tensor_model_parallel_size=world)
    g = ps.get_tensor_model_parallel_group()
    ws = _fused_impl.workspace(g)
    S, H, I, V = 4096, 4096, 11008, 32000
    peaks = json.load(open("MEASURED_PEAKS.json")) if os.path.exists("MEASURED_PEAKS.json") else {}
    peak_tf = peaks.get("bf16_tflops", 1590.0)
    link_gbs = 770.0
    res = []

    def report(name, M, N, K, wire_bytes, fused, base_own, base_lib):
        flops = 2.0 * M * N * K
        roof_us = max(flops / (peak_tf * 1e12), wire_bytes / (link_gbs * 1e9)) * 1e6
        r = {"op": name, "M": M, "N": N, "K": K, "tp": world, "fused_us": fused, "nccl_plus_own_gemm_us": base_own,
             "nccl_plus_cublas_us": base_lib, "roofline_us": roof_us, "fraction_of_roofline": roof_us / fused,
             "bound": "compute" if flops / (peak_tf * 1e12) > wire_bytes / (link_gbs * 1e9) else "nvlink"}
        res.append(r)
        if rank == 0:
            print(json.dumps(r), flush=True)

    for name, N in (("ag_gemm_qkv", 3 * H // world), ("ag_gemm_gate_up", 2 * I // world), ("ag_gemm_lm_head", V // world)):
        x = torch.randn(S // world, H, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(N, H, device="cuda", dtype=torch.bfloat16)
        fused = timeit(lambda: ws.ag_gemm(x, w, True))
        own = timeit(lambda: gemm.matmul(comm.all_gather(x, 0, g), w, False, True))
        lib = timeit(lambda: torch.matmul(comm.all_gather(x, 0, g), w.t()))
        report(name, S, N, H, (world - 1) * x.numel() * 2, fused, own, lib)
    for name, K in (("gemm_rs_o_proj", H // world), ("gemm_rs_down", I // world)):
        x = torch.randn(S, K, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(H, K, device="cuda", dtype=torch.bfloat16)
        fused = timeit(lambda: ws.gemm_rs(x, w, True))
        own = timeit(lambda: comm.reduce_scatter(gemm.matmul(x, w, False, True), 0, g))
        lib = timeit(lambda: comm.reduce_scatter(torch.matmul(x, w.t()), 0, g))
        report(name, S, H, K, (world - 1) * (S // world) * H * 2, fused, own, lib)
    # optional sweep: comm-CTA split × micro-batch rows (fused kernels only)
    if "--sweep" in sys.argv:
        sweep = []
        comm_sms0, nvls_config0 = _fused_impl._COMM_SMS, dict(_fused_impl.NVLS_CONFIG)
        for M in (4096, 16384):
            if (M // world) % 256 or M // world // 128 > 64:
                continue
            for ag, rs in ((12, 16), (24, 24), (32, 32)):
                # cudaIpc kernels take the all-gather split from _COMM_SMS, the NVLS kernels both splits from NVLS_CONFIG
                _fused_impl._COMM_SMS = _fused_impl.NVLS_CONFIG["comm_ctas_ag"] = ag
                _fused_impl.NVLS_CONFIG["comm_ctas_rs"] = rs
                x = torch.randn(M // world, H, device="cuda", dtype=torch.bfloat16)
                w = torch.randn(2 * I // world, H, device="cuda", dtype=torch.bfloat16)
                t_ag = timeit(lambda: ws.ag_gemm(x, w, True), iters=10, warmup=3)
                x2 = torch.randn(M, I // world, device="cuda", dtype=torch.bfloat16)
                w2 = torch.randn(H, I // world, device="cuda", dtype=torch.bfloat16)
                t_rs = timeit(lambda: ws.gemm_rs(x2, w2, True), iters=10, warmup=3)
                rec = {"sweep": True, "M": M, "comm_ctas_ag": ag, "comm_ctas_rs": rs, "ag_gemm_gate_up_us": t_ag, "gemm_rs_down_us": t_rs}
                sweep.append(rec)
                if rank == 0:
                    print(json.dumps(rec), flush=True)
        _fused_impl._COMM_SMS, _fused_impl.NVLS_CONFIG = comm_sms0, nvls_config0
        res.append({"sweep": sweep})
    # raw collectives for reference
    x = torch.randn(S // world, H, device="cuda", dtype=torch.bfloat16)
    y = torch.randn(S, H, device="cuda", dtype=torch.bfloat16)
    extra = {"nccl_all_gather_us": timeit(lambda: comm.all_gather(x, 0, g)),
             "nccl_reduce_scatter_bf16_us": timeit(lambda: comm.reduce_scatter(y, 0, g)),
             "nccl_reduce_scatter_fp32_us": timeit(lambda: comm.reduce_scatter(y.float(), 0, g))}
    if rank == 0:
        print(json.dumps(extra), flush=True)
        os.makedirs("gpurun_out", exist_ok=True)
        json.dump({"ops": res, "collectives": extra}, open(f"gpurun_out/tp_bench_tp{world}.json", "w"), indent=1)
    dist.barrier()
    ps.destroy_model_parallel()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
