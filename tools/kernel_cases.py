"""Isolated launches of every kernel mode through the C-ABI stager seam, for ncu captures and CUDA-event roofline
numbers:  dense (bulk/TMA), column shard (rows/TMA), odd-alignment slab member (LSU contig), transpose (LSU tiled),
fp32->bf16, fp32->e4m3fn and bf16->e4m3fn casts (LSU cast), short strided runs (LSU strided), per-channel int8 quantisation (statistics + parameters +
quantising pack) along dim 0 and dim 1, its dequantising scatter, the same for per-channel scaled float8 (fp8chan_*), and an
e4m3fn -> bf16 converting scatter.  Prints one JSON line per case with the kernel's
CUDA-event time and achieved GB/s against the measured HBM copy peak (MEASURED_PEAKS.json; else the H100 SXM data
sheet's 3.35 TB/s).  A per-channel save reads its source twice (statistics, then the pack): its algorithmic bytes are
both reads, the 1-byte elements written and the 16 (int8) or 4 (float8) bytes of parameters per channel; a dequantising
restore's the 1-byte elements read, the parameters and the target written; a cast's are the source and destination
element sizes per element.

    python tools/kernel_cases.py [--case NAME_OR_GLOB] [--reps N]      (e.g. --case 'fp8chan_*')
    ncu --set full --clock-control none --import-source on -k regex:tsnap -o kernels python tools/kernel_cases.py --reps 1
"""
import argparse, fnmatch, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from torchsnapshot_b200 import _native as N

ap = argparse.ArgumentParser(); ap.add_argument("--case", default="all"); ap.add_argument("--reps", type=int, default=5); args = ap.parse_args()
dev = "cuda:0"
eng = N.Engine(device=0, io_threads=2, pinned_slot_bytes=32 << 20, pinned_slots=4)
try:
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    peak = 3350.0

def cases():
    GiB = 1 << 30
    base = torch.empty(GiB // 4, dtype=torch.float32, device=dev).uniform_()  # 1 GiB
    yield "dense_bulk_1GiB", [(base, 0, None)], GiB, 2 * GiB
    wide = base.view(1 << 20, 256)
    v = wide[:, 64:192]  # 512 B runs, 1 KiB pitch
    yield "column_shard_512B_runs", [(v, 0, None)], v.numel() * 4, 2 * v.numel() * 4
    w4k = base.view(1 << 16, 4096)[:, 1024:3072]  # 8 KiB runs, 16 KiB pitch
    yield "column_shard_8KiB_runs", [(w4k, 0, None)], w4k.numel() * 4, 2 * w4k.numel() * 4
    yield "odd_alignment_contig_1GiB", [(base[:-4], 3, None)], GiB, 2 * (GiB - 16)
    sq = base[: 8192 * 8192].view(8192, 8192).t()
    yield "transpose_fp32_8192x8192", [(sq, 0, None)], sq.numel() * 4, 2 * sq.numel() * 4
    hb = base.view(torch.bfloat16)[: 16384 * 8192].view(16384, 8192).t()
    yield "transpose_bf16_16384x8192", [(hb, 0, None)], hb.numel() * 2, 2 * hb.numel() * 2
    yield "cast_fp32_to_bf16_1GiB", [(base, 0, torch.bfloat16)], GiB // 2, GiB + GiB // 2
    yield "cast_fp32_to_e4m3fn_1GiB", [(base, 0, torch.float8_e4m3fn)], GiB // 4, GiB + GiB // 4
    hb = base.view(torch.bfloat16)
    yield "cast_bf16_to_e4m3fn_1GiB", [(hb, 0, torch.float8_e4m3fn)], GiB // 2, GiB + GiB // 2
    short = base.view(1 << 22, 64)[:, 8:40]  # 128 B runs: below the copy-engine threshold
    yield "strided_128B_runs", [(short, 0, None)], short.numel() * 4, 2 * short.numel() * 4
    m = base.view(262144, 1024)
    for axis in (0, 1):
        C = m.shape[axis]
        yield f"qchannel_fp32_axis{axis}_1GiB", [(m, 8, torch.qint8, axis)], 8 + m.numel() + 16 * C, 2 * GiB + m.numel() + 16 * C
    hb = torch.empty(524288, 1024, dtype=torch.bfloat16, device=dev).normal_()  # finite values (reinterpreted fp32 bits are not)
    yield "qchannel_bf16_axis0_1GiB", [(hb, 8, torch.qint8, 0)], 8 + hb.numel() + 16 * 524288, 2 * GiB + hb.numel() + 16 * 524288
    for fmt, fp8 in (("e4m3fn", torch.float8_e4m3fn), ("e5m2", torch.float8_e5m2)):
        for axis in (0, 1):
            C = m.shape[axis]
            yield f"fp8chan_{fmt}_fp32_axis{axis}_1GiB", [(m, 8, fp8, axis)], 8 + m.numel() + 4 * C, 2 * GiB + m.numel() + 4 * C
        yield f"fp8chan_{fmt}_bf16_axis0_1GiB", [(hb, 8, fp8, 0)], 8 + hb.numel() + 4 * 524288, 2 * GiB + hb.numel() + 4 * 524288

def selected(name):
    return args.case == "all" or fnmatch.fnmatch(name, args.case)


for name, members, nbytes, algo in cases():
    if not selected(name):
        continue
    descs = [N.save_desc(m[0], m[1], wire_dtype=m[2], axis=m[3] if len(m) > 3 else None) for m in members]
    total = nbytes + 16
    best = None
    for rep in range(args.reps + 1):
        sb = eng.stage(descs, total, stream=torch.cuda.current_stream().cuda_stream, keepalive=[m[0] for m in members])
        sb.wait(); st = sb.stats(); sb.release()
        if rep and (best is None or st["kernel_ms"] < best["kernel_ms"]):
            best = st
    st = best or st
    print(json.dumps({"case": name, "kernel_ms": round(st["kernel_ms"], 4), "bulk_ms": round(st["kernel_bulk_ms"], 4), "rows_ms": round(st["kernel_rows_ms"], 4),
                      "lsu_ms": round(st["kernel_lsu_ms"], 4), "tiles": [st["n_tiles_bulk"], st["n_tiles_rows"], st["n_tiles_lsu"]],
                      "algorithmic_bytes": algo, "gbs": round(algo / 1e6 / st["kernel_ms"], 1), "frac_of_measured_peak": round(algo / 1e6 / st["kernel_ms"] / peak, 3)}), flush=True)

# dequantising scatter: the [262144, 1024] target of an axis-0 per-channel image already in device memory
def dequant_case(name, wire_dtype, pbytes, target):
    dst = torch.empty(262144, 1024, dtype=target, device=dev)
    wire = torch.empty(8 + dst.numel() + pbytes * 262144, dtype=torch.uint8, device=dev)
    sb = eng.stage([N.save_desc(dst.uniform_(), 8, wire_dtype=wire_dtype, axis=0)], wire.numel(), keepalive=[dst])
    wire.copy_(torch.frombuffer(bytearray(sb.wait()), dtype=torch.uint8).to(dev)); sb.release()
    desc = N.per_channel(N.load_desc(dst, 8, wire_dtype=wire_dtype), [262144, 1024], 0, 8)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for rep in range(args.reps + 1):
        ev[0].record(); eng.scatter_device(wire, [desc]); ev[1].record(); torch.cuda.synchronize()
        if rep:
            times.append(ev[0].elapsed_time(ev[1]))
    ms = min(times)
    algo = dst.numel() + pbytes * 262144 + dst.numel() * dst.element_size()
    print(json.dumps({"case": name, "kernel_ms": round(ms, 4), "note": "CUDA events around tsnap_scatter_device (table upload + launch + kernel)",
                      "algorithmic_bytes": algo, "gbs": round(algo / 1e6 / ms, 1), "frac_of_measured_peak": round(algo / 1e6 / ms / peak, 3)}), flush=True)


for name, wire_dtype, pbytes, target in (
    ("qchannel_dequant_fp32_axis0_1GiB", torch.qint8, 16, torch.float32),
    ("fp8chan_e4m3fn_dequant_fp32_axis0_1GiB", torch.float8_e4m3fn, 4, torch.float32),
    ("fp8chan_e4m3fn_dequant_bf16_axis0", torch.float8_e4m3fn, 4, torch.bfloat16),
    ("fp8chan_e5m2_dequant_fp32_axis0_1GiB", torch.float8_e5m2, 4, torch.float32),
    ("fp8chan_e5m2_dequant_bf16_axis0", torch.float8_e5m2, 4, torch.bfloat16),
):
    if selected(name):
        dequant_case(name, wire_dtype, pbytes, target)
# converting scatter: a 1 GiB bf16 target from an e4m3fn image already in device memory
if selected("scatter_e4m3fn_to_bf16_1GiB"):
    dst = torch.empty(1 << 29, dtype=torch.bfloat16, device=dev)
    wire = torch.empty(1 << 29, dtype=torch.float8_e4m3fn, device=dev).view(torch.uint8).random_(0, 256)
    desc = N.load_desc(dst, 0, wire_dtype=torch.float8_e4m3fn)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for rep in range(args.reps + 1):
        ev[0].record(); eng.scatter_device(wire, [desc]); ev[1].record(); torch.cuda.synchronize()
        if rep:
            times.append(ev[0].elapsed_time(ev[1]))
    ms = min(times)
    algo = dst.numel() * 3
    print(json.dumps({"case": "scatter_e4m3fn_to_bf16_1GiB", "kernel_ms": round(ms, 4), "note": "CUDA events around tsnap_scatter_device (table upload + launch + kernel)",
                      "algorithmic_bytes": algo, "gbs": round(algo / 1e6 / ms, 1), "frac_of_measured_peak": round(algo / 1e6 / ms / peak, 3)}), flush=True)
eng.close()
