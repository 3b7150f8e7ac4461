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

    python tools/bench_detector.py [--precision exact] [--frames 200] [--warmup 20] [--reps 20] [--rounds 1] [--cpu-frames 2]
                                   [--out file.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-frames", type=int, default=2)
    ap.add_argument("--nets", default="yolov2-tiny,yolov3")
    ap.add_argument("--precision", default="exact", help="comma-separated: exact, tf32")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from ground_fusion_b200.synth import SyntheticStream
    st = SyntheticStream(seed=0)
    frames = [np.ascontiguousarray(st.color(k)[..., ::-1]) for k in range(8)]
    gpu = gpu_name_and_power_limit()
    with tempfile.TemporaryDirectory() as tmp:
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
