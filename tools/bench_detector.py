"""Throughput of the YOLO detector (gf_detector) for yolov2-tiny and yolov3 at their shipped 416x416, from 640x480 BGR8 host
frames, with seeded weights (tests/yolo_ref.write_weights; the arithmetic, not the weights' values, sets the time).

Prints one JSON line (and writes it to --out): per network
  - detections/s: wall clock over --frames calls of YoloDetector.detect (upload, letterbox, graph, decoding, NMS, extraction),
    after --warmup calls;
  - device_ms: gf_detector_last_device_ms (CUDA events around letterbox + graph), median over the same calls;
  - per-layer kernel time: CUDA events around each layer's kernels re-run --reps times (gf_detector_layer_times);
  - conv FLOP/s: 2 M N K per convolution over the summed convolution time, against the bound of the precision's arithmetic.
    exact: sequential FMUL + FADD chains (no FMA, no tensor cores, to stay bit-exact with darknet), so the bound is half of
    the data sheet's 67 TFLOP/s FP32 FFMA rate: 33.5 TFLOP/s.  tf32: the data sheet's 495 TFLOP/s dense TF32 tensor-core
    rate (H100 SXM, a data-sheet figure, not a measurement);
  - host_ms_per_call: wall time per call minus the median device time (frame upload, decoding, NMS, extraction, Python);
  - the single-thread darknet CPU oracle on the same host over --cpu-frames frames, when it is built.
With --precision exact,tf32 both precisions are timed in the same run on the same card, alternating per network in blocks of
--frames calls (--rounds rounds; the medians over rounds are reported).  The card's name and power limit are read in the same run.

With --batch 1,2,4,8,16 it times gf_detector_detect_batch instead, for each network, precision and n, on one handle sized for
the largest n: --batch-calls calls of detect_batch over n distinct 640x480 frames, alternating in each round with the same n
frames through n sequential detect calls on the same handle.  Per n: device ms per call (CUDA events around letterbox + graph;
for the sequential form the sum of its n calls), host ms per call (wall time minus device time), frames per second in total,
the per-frame gain of the batch over the sequential calls, and per layer the batch's time over n times one frame's
(gf_detector_layer_times), which names the layers where a batch is not faster.  The handle's device memory (cudaMemGetInfo
before and after creating it and sizing it) is reported per network and precision.

    python tools/bench_detector.py [--precision exact] [--frames 200] [--warmup 20] [--reps 20] [--rounds 1] [--cpu-frames 2]
                                   [--batch 1,2,4,8,16 --batch-calls 30] [--out file.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

from ground_fusion_b200.detector import YoloDetector, parse_cfg  # noqa: E402
import yolo_ref  # noqa: E402

FMUL_FADD_BOUND = 67e12 / 2
TF32_DATA_SHEET = 495e12
BOUNDS = {"exact": ("FMUL + FADD: half of the H100 SXM data sheet's 67 TFLOP/s FP32 FFMA rate = 33.5 TFLOP/s", FMUL_FADD_BOUND),
          "tf32": ("TF32 tensor cores: the H100 SXM data sheet's 495 TFLOP/s dense TF32 rate", TF32_DATA_SHEET)}


def gpu_name_and_power_limit():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                       text=True).strip()
    except Exception as e:   # the measurement still needs a device; only the label is missing
        return "unknown (%s)" % e


def conv_flops(cfg):
    _, layers = parse_cfg(cfg)
    return [2.0 * L["n"] * L["out_w"] * L["out_h"] * L["c"] * L["size"] ** 2 if L["type"] == "convolutional" else 0.0
            for L in layers], layers


def timed_block(det, args, frames):
    """--frames calls after --warmup: (wall seconds, device ms of each call, per-layer ms)."""
    for k in range(args.warmup):
        det.detect(frames[k % len(frames)])
    dev = []
    t0 = time.perf_counter()
    for k in range(args.frames):
        det.detect(frames[k % len(frames)])
        dev.append(det.last_device_ms())
    wall = time.perf_counter() - t0
    return wall, dev, det.layer_times(args.reps)


def result(name, precision, flops, layers, args, blocks):
    walls = [b[0] for b in blocks]
    dev = [float(np.median(b[1])) for b in blocks]
    per_layer = np.median(np.stack([b[2] for b in blocks]), axis=0)
    conv_ms = float(sum(per_layer[i] for i, f in enumerate(flops) if f))
    total = sum(flops)
    bound = BOUNDS[precision][1]
    tf = total / (conv_ms * 1e-3)
    out = {"net": name, "precision": precision, "net_size": [416, 416], "frame": [640, 480],
           "detections_per_s": args.frames / float(np.median(walls)),
           "device_ms_median": float(np.median(dev)), "layers_ms_sum": float(per_layer.sum()), "conv_ms_sum": conv_ms,
           "host_ms_per_call": float(np.median(walls)) / args.frames * 1e3 - float(np.median(dev)),
           "conv_gflop": total / 1e9, "conv_tflops": tf / 1e12, "bound": BOUNDS[precision][0],
           "conv_share_of_bound": tf / bound, "conv_floor_ms_at_bound": total / bound * 1e3,
           "per_layer": [{"i": i, "type": L["type"], "out": [L["out_c"], L["out_h"], L["out_w"]], "ms": round(float(per_layer[i]), 5),
                          "gflop": round(flops[i] / 1e9, 4)} for i, L in enumerate(layers)]}
    if precision == "exact":
        out["conv_share_of_fmul_fadd_bound"] = out["conv_share_of_bound"]
    for e in out["per_layer"]:
        if e["gflop"] > 0 and e["ms"] > 0:
            e["tflops"] = round(e["gflop"] / e["ms"], 3)
            e["share_of_bound"] = round(e["gflop"] * 1e9 / (e["ms"] * 1e-3) / bound, 4)
    return out


def run(name, tmp, args, frames):
    """One network at every requested precision: one detector per precision, timed in alternating blocks."""
    cfg = yolo_ref.cfg_path(name)
    w = yolo_ref.write_weights(cfg, os.path.join(tmp, name + ".weights"), seed=1)
    flops, layers = conv_flops(cfg)
    precisions = args.precision.split(",")
    dets = {p: YoloDetector(cfg, w, thresh=0.3, precision=p) for p in precisions}
    blocks = {p: [] for p in precisions}
    try:
        for _ in range(args.rounds):
            for p in precisions:
                blocks[p].append(timed_block(dets[p], args, frames))
    finally:
        for d in dets.values():
            d.close()
    outs = [result(name, p, flops, layers, args, blocks[p]) for p in precisions]
    if "exact" in blocks and "tf32" in blocks:
        ex, tf = outs[precisions.index("exact")], outs[precisions.index("tf32")]
        tf["conv_ms_ratio_to_exact"] = tf["conv_ms_sum"] / ex["conv_ms_sum"]
        tf["device_ms_ratio_to_exact"] = tf["device_ms_median"] / ex["device_ms_median"]
    out = outs[0] if len(outs) == 1 else {"net": name, "precisions": outs}
    if args.cpu_frames > 0 and yolo_ref.oracle_available():
        ref = yolo_ref.Darknet(cfg, w)
        try:
            t0 = time.perf_counter()
            for k in range(args.cpu_frames):
                ref.detect(frames[k % len(frames)], 0.3)
            out["cpu_oracle_s_per_frame"] = (time.perf_counter() - t0) / args.cpu_frames
        finally:
            ref.close()
    return out


def device_free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def batch_block(det, frames, calls):
    """calls x detect_batch(frames), then calls x (one detect per frame): per form (wall s per call, median device ms per call)."""
    det.detect_batch(frames)
    dev_b = []
    t0 = time.perf_counter()
    for _ in range(calls):
        det.detect_batch(frames)
        dev_b.append(det.last_device_ms())
    wall_b = (time.perf_counter() - t0) / calls
    for f in frames:
        det.detect(f)
    dev_s = []
    t0 = time.perf_counter()
    for _ in range(calls):
        ms = 0.0
        for f in frames:
            det.detect(f)
            ms += det.last_device_ms()
        dev_s.append(ms)
    wall_s = (time.perf_counter() - t0) / calls
    return (wall_b, float(np.median(dev_b))), (wall_s, float(np.median(dev_s)))


def run_batch(name, tmp, args, frames):
    """One network: per precision one handle sized for the largest n, every n timed in alternating batch / sequential blocks."""
    cfg = yolo_ref.cfg_path(name)
    w = yolo_ref.write_weights(cfg, os.path.join(tmp, name + ".weights"), seed=1)
    _, layers = conv_flops(cfg)
    ns = [int(v) for v in args.batch.split(",")]
    out = {"net": name, "net_size": [416, 416], "frame": [640, 480], "precisions": []}
    for p in args.precision.split(","):
        free0 = device_free_bytes()
        det = YoloDetector(cfg, w, thresh=0.3, precision=p)
        free1 = device_free_bytes()
        det.set_max_batch(max(ns))
        free2 = device_free_bytes()
        res = {"precision": p, "handle_mib_at_max_batch_1": (free0 - free1) / 2 ** 20,
               "handle_mib_at_max_batch_%d" % max(ns): (free0 - free2) / 2 ** 20, "batches": []}
        try:
            blocks = {n: [] for n in ns}
            for _ in range(args.rounds):
                for n in ns:
                    blocks[n].append(batch_block(det, frames[:n], args.batch_calls))
            for n in ns:
                (wb, db), (ws, ds) = [(float(np.median([b[k][0] for b in blocks[n]])), float(np.median([b[k][1] for b in blocks[n]])))
                                      for k in (0, 1)]
                det.detect(frames[0])
                one = det.layer_times(args.reps)
                det.detect_batch(frames[:n])
                many = det.layer_times(args.reps)
                ratio = many / np.maximum(n * one, 1e-9)
                slow = [{"i": int(i), "type": layers[i]["type"], "out": [layers[i]["out_c"], layers[i]["out_h"], layers[i]["out_w"]],
                         "batch_ms": round(float(many[i]), 5), "n_x_single_ms": round(float(n * one[i]), 5),
                         "ratio": round(float(ratio[i]), 3)} for i in np.argsort(-ratio)[:5]]
                res["batches"].append({
                    "n": n, "batch_device_ms": db, "batch_host_ms": wb * 1e3 - db, "batch_fps": n / wb,
                    "sequential_device_ms": ds, "sequential_host_ms": ws * 1e3 - ds, "sequential_fps": n / ws,
                    "device_gain_per_frame": ds / db, "wall_gain_per_frame": ws / wb,
                    "layers_ms_batch": float(many.sum()), "layers_ms_n_x_single": float(n * one.sum()),
                    "layers_least_gain": slow})
        finally:
            det.close()
        out["precisions"].append(res)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-frames", type=int, default=2)
    ap.add_argument("--nets", default="yolov2-tiny,yolov3")
    ap.add_argument("--precision", default="exact", help="comma-separated: exact, tf32")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--batch", default=None, help="comma-separated batch sizes: time detect_batch against sequential detect")
    ap.add_argument("--batch-calls", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from ground_fusion_b200.synth import SyntheticStream
    st = SyntheticStream(seed=0)
    n_frames = max([8] + [int(v) for v in args.batch.split(",")] if args.batch else [8])
    frames = [np.ascontiguousarray(st.color(k)[..., ::-1]) for k in range(n_frames)]
    gpu = gpu_name_and_power_limit()
    with tempfile.TemporaryDirectory() as tmp:
        if args.batch:
            res = {"gpu": gpu, "rounds": args.rounds, "calls_per_block": args.batch_calls,
                   "nets": [run_batch(n, tmp, args, frames) for n in args.nets.split(",")]}
        else:
            res = {"gpu": gpu, "nets": [run(n, tmp, args, frames) for n in args.nets.split(",")]}
            if args.precision == "exact":
                res["bound"] = BOUNDS["exact"][0]
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
