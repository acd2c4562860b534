"""Per-channel int8 quantise-on-save, per-channel scaled float8 and the e4m3fn cast on the C3 checkpoint (FSDP-layout
Llama-3-8B bf16, one rank: 291 tensors, 16.06 GB).

For each of two alternating rounds, and for the plain snapshot, ``quantize_on_save(torch.qint8, axis=0)``,
``quantize_on_save(torch.float8_e4m3fn, axis=0)`` and ``cast_on_save(torch.float8_e4m3fn)``:
``Snapshot.take`` and ``restore`` wall time, bytes on disk, and how long ``async_take`` blocks the caller.  The card's
name and power limit are read in the same run.  Prints one JSON line per (round, variant) and a summary line.

    python tools/quant_take.py [--dir DIR] [--rounds 2]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import torchsnapshot_b200 as B  # noqa: E402
from benchmarks import workloads as W  # noqa: E402


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["sm_max_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001
        out["power_limit"] = f"unavailable ({e})"
    return out


def du(path: str) -> int:
    return sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(path) for f in fs)


def timed(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=os.environ.get("TSNAP_BENCH_DIR"))
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("quant_take.py measures on the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    store = tempfile.NamedTemporaryFile(delete=False)
    dist.init_process_group("gloo", init_method=f"file://{store.name}", rank=0, world_size=1)
    base = tempfile.mkdtemp(prefix="tsnap_quant_", dir=args.dir)
    try:
        local = W.build_llama_local(0, 1, dev)
        app = {"model": B.StateDict(**W.wrap_sharded(local, 0, dev))}
        payload = sum(t.numel() * t.element_size() for t, _, _ in local.values())
        info = card()
        hooks = {"plain": None, "qint8_axis0": B.quantize_on_save(torch.qint8, axis=0),
                 "e4m3fn_axis0": B.quantize_on_save(torch.float8_e4m3fn, axis=0), "e4m3fn_cast": B.cast_on_save(torch.float8_e4m3fn)}
        for name, hook in hooks.items():  # warm-up: module loads, the arena, the pinned ring
            B.Snapshot.take(os.path.join(base, "warm"), app, _custom_tensor_prepare_func=hook)
            shutil.rmtree(os.path.join(base, "warm"))
        results = []
        for r in range(args.rounds):
            for name, hook in hooks.items():
                path = os.path.join(base, f"{name}{r}")
                take_ms = timed(lambda: B.Snapshot.take(path, app, _custom_tensor_prepare_func=hook))
                on_disk = du(path)
                restore_ms = timed(lambda: B.Snapshot(path).restore(app))
                shutil.rmtree(path)
                t0 = time.perf_counter()
                pending = B.Snapshot.async_take(path, app, _custom_tensor_prepare_func=hook)
                block_ms = (time.perf_counter() - t0) * 1e3
                pending.wait()
                shutil.rmtree(path)
                line = {"round": r, "variant": name, "take_ms": round(take_ms, 1), "restore_ms": round(restore_ms, 1),
                        "async_take_block_ms": round(block_ms, 1), "bytes_on_disk": on_disk, "payload_bytes": payload,
                        "take_gbs_of_payload": round(payload / 1e6 / take_ms, 2), "card": info}
                results.append(line)
                print(json.dumps(line), flush=True)
        summary = {}
        for name in hooks:
            rows = [x for x in results if x["variant"] == name]
            summary[name] = {k: [x[k] for x in rows] for k in ("take_ms", "restore_ms", "async_take_block_ms", "bytes_on_disk")}
        print(json.dumps({"summary": summary, "card": info, "workload": "C3 N=1: FSDP-layout Llama-3-8B bf16, ShardedTensor per weight"}), flush=True)
    finally:
        shutil.rmtree(base, ignore_errors=True)
        dist.destroy_process_group()
        os.unlink(store.name)


if __name__ == "__main__":
    main()
