#!/usr/bin/env python
"""Steady-state per-pass kernel times of the bench.py workload (REBLUR_DIFFUSE_SPECULAR, 3840x2160, default settings) and byte
digests of what temporal accumulation writes, for A/B comparisons of builds of the library.

bench.py's per-pass breakdown replays the last frames on top of the history of the final one, so the motion vectors of the first
replayed frame point at a history that is several frames newer: most pixels are disoccluded and the temporal passes run their
young-history paths.  Here every frame is denoised once, in order, and each dispatch is timed with the executor's own events
(nrdCudaSetTiming: kernel time only), so the numbers are what a running application pays per frame.

    python tools/time_reblur_passes.py [--frames 24 --warmup 6]                  one library (NRD_B200_LIB, else the in-tree build)
    python tools/time_reblur_passes.py --ab parent=LIB_A new=LIB_B [--rounds 3] [--bench-steps 24] [--out FILE.json]

--ab runs one process per library and round, alternating the libraries (the first one is the baseline), and compares the digests
of every frame with the baseline's.  --bench-steps also alternates `bench.py` runs of each library.  A GPU is required.

The digests copy every texture temporal accumulation writes and reduce it on the GPU before HistoryFix runs, which changes what
HistoryFix finds in L2 (temporal accumulation itself is timed before the copies).  --no-digest times the passes without them.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
        name, power, max_sm = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": max_sm}
    except Exception as e:  # the numbers are still printed, marked as unattributed
        return {"gpu": "unknown (%s)" % e}


class Digests(object):
    """Byte digests of textures, reduced on the GPU: the sum of the 32-bit words, and two sums weighted by the word index."""

    def __init__(self, ctx, stream):
        self.ctx, self.stream, self.weights, self.staging = ctx, stream, {}, {}

    def tensor(self, t):
        import torch
        v = t.contiguous().view(torch.uint8).reshape(-1).view(torch.int32).to(torch.int64)
        if v.numel() not in self.weights:
            i = torch.arange(v.numel(), device=v.device, dtype=torch.int64)
            self.weights[v.numel()] = ((i % 8191) + 1, (i % 65521) + 1)
        w1, w2 = self.weights[v.numel()]
        return torch.stack([v.sum(), (v * w1).sum(), (v * w2).sum()])

    def texture(self, rtype, index):
        # the texel bytes of the rows the context holds, copied into a buffer of the texture's pitch (padding stays zero)
        import torch
        info = self.ctx.get_texture(rtype, index)
        key = (int(rtype), index)
        if key not in self.staging:
            self.staging[key] = torch.zeros((info.rowsNum * info.pitchBytes + 3) // 4 * 4, dtype=torch.uint8, device=self.stream.device)
        self.ctx.copy(rtype, index, self.staging[key].data_ptr(), info.pitchBytes, False, self.stream.cuda_stream)
        return self.tensor(self.staging[key])

    @staticmethod
    def hex(digests):
        return {k: "%x.%x.%x" % tuple(int(x) & (2 ** 64 - 1) for x in v.cpu().tolist()) for k, v in digests.items()}


def worker(args):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_reblur_passes.py needs a CUDA device")
    from bench import ClockSampler
    from raytracingdenoiser_b200 import harness, nrd, scene
    W, H = args.width, args.height
    den = nrd.Denoiser.REBLUR_DIFFUSE_SPECULAR
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    sc = scene.Scene(W, H, device="cuda:0")
    gpu = harness.GpuDenoiser(den, W, H)
    ctx, inst = gpu.ctx, gpu.instance
    pipelines = inst.get_instance_desc()["pipelines"]
    dg = Digests(ctx, stream)
    sampler = ClockSampler(0)
    ctx.set_timing(True)
    per_pass, frame_digests, frame_ms = {}, [], []
    for i in range(args.warmup + args.frames):
        if i == args.warmup:
            torch.cuda.synchronize()
            sampler.start()
        fr = sc.frame(i)
        gpu.set_inputs(fr)
        inst.set_common_settings(harness.make_common_settings(fr, W, H, i))
        r, raw, n = inst.get_compute_dispatches_raw([gpu.identifier])
        if r != nrd.Result.SUCCESS:
            raise RuntimeError("GetComputeDispatches: %s" % r)
        dispatches = [nrd.Dispatch(raw[j], pipelines) for j in range(n)]
        ctx.barrier(stream.cuda_stream)  # what nrdCudaDenoise does at the start of a frame
        names, digests = [], {}
        for j in range(n):
            ctx.execute_raw(C.byref(raw[j]), stream.cuda_stream)
            name = dispatches[j].name.split(" - ")[-1]
            if dispatches[j].shaderFileName.startswith("Clear_"):  # clears are not timed (executor.cu)
                continue
            names.append(name)
            if name == "Temporal accumulation" and not args.no_digest:
                for dt, rt, idx in dispatches[j].resources:
                    if dt == nrd.DescriptorType.STORAGE_TEXTURE:
                        digests["TA:%s[%d]" % (rt.name, idx)] = dg.texture(rt, idx)
        for name, t in sorted(gpu.outputs().items()):
            if not args.no_digest:
                digests[name] = dg.tensor(t)
        kernel_ms, _ = ctx.get_timing()  # synchronises
        frame_digests.append(Digests.hex(digests))
        if len(kernel_ms) != len(names):
            raise RuntimeError("%d timed dispatches for %d dispatch names" % (len(kernel_ms), len(names)))
        if i >= args.warmup:
            this_frame = {}
            for name, ms in zip(names, kernel_ms):
                this_frame[name] = this_frame.get(name, 0.0) + ms
            for name, ms in this_frame.items():
                per_pass.setdefault(name, []).append(ms)
            frame_ms.append(sum(kernel_ms))
    clocks = sampler.stop()
    ctx.set_timing(False)
    gpu.destroy()
    out = {"lib": os.environ.get("NRD_B200_LIB", "in-tree"), "size": [W, H], "warmup": args.warmup, "frames": args.frames, "digests_recorded": not args.no_digest,
           "median_ms": {k: statistics.median(v) for k, v in per_pass.items()}, "frame_ms_median": statistics.median(frame_ms),
           "ta_ms": per_pass["Temporal accumulation"], "clocks": clocks, "digests": frame_digests}
    out.update(gpu_info())
    print("RESULT " + json.dumps(out))


def run_worker(lib, args):
    env = dict(os.environ, NRD_B200_LIB=os.path.abspath(lib))
    cmd = [sys.executable, os.path.abspath(__file__), "--frames", str(args.frames), "--warmup", str(args.warmup), "--width", str(args.width), "--height", str(args.height)]
    cmd += ["--no-digest"] if args.no_digest else []
    r = subprocess.run(cmd, env=env, capture_output=True, text=True)
    for line in r.stdout.splitlines():
        if line.startswith("RESULT "):
            return json.loads(line[7:])
    raise RuntimeError("worker for %s failed (exit %d):\n%s%s" % (lib, r.returncode, r.stdout[-3000:], r.stderr[-3000:]))


def run_bench(lib, args, dump_dir):
    env = dict(os.environ, NRD_B200_LIB=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps), "--warmup", "6", "--no-cpu-baseline", "--dump-outputs", dump_dir]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError("bench.py with %s failed (exit %d):\n%s" % (lib, r.returncode, r.stderr[-3000:]))
    return json.loads(lines[-1])


def same_files(a, b):
    import numpy as np
    names = sorted(os.listdir(a))
    return names == sorted(os.listdir(b)) and all(np.array_equal(np.load(os.path.join(a, n)), np.load(os.path.join(b, n))) for n in names)


def driver(args):
    import tempfile
    libs = [x.split("=", 1) for x in args.ab]
    results = {name: [] for name, _ in libs}
    benches = {name: [] for name, _ in libs}
    report = {"gpu": gpu_info(), "rounds": args.rounds, "frames": args.frames, "warmup": args.warmup}
    print(json.dumps(report["gpu"]), flush=True)
    dumps = tempfile.mkdtemp(prefix="nrd_ab_")
    mismatches = {}
    for rnd in range(args.rounds):
        for name, lib in libs:
            res = run_worker(lib, args)
            results[name].append(res)
            base = results[libs[0][0]][rnd]
            bad = [(f, k) for f, (d0, d1) in enumerate(zip(base["digests"], res["digests"])) for k in d0 if d0[k] != d1.get(k)]
            if res["digests"] != results[name][0]["digests"]:
                bad.append(("run-to-run", "digests differ between rounds of the same build"))
            mismatches.setdefault(name, []).extend(bad)
            print("round %d %-8s TA median %.4f ms  frame (sum of kernels) %.4f ms  sm %s MHz  digest mismatches vs %s: %s" % (
                rnd, name, res["median_ms"]["Temporal accumulation"], res["frame_ms_median"], res["clocks"]["sm_mhz"], libs[0][0],
                "not recorded" if args.no_digest else len(bad)), flush=True)
        if args.bench_steps:
            for name, lib in libs:
                b = run_bench(lib, args, os.path.join(dumps, "%s_%d" % (name, rnd)))
                benches[name].append(b["value"])
                print("round %d %-8s bench.py value %.1f Mpixels/s  sm %s MHz" % (rnd, name, b["value"], (b.get("clocks") or {}).get("sm_mhz")), flush=True)
    summary = {}
    for name, _ in libs:
        tas = [r["median_ms"]["Temporal accumulation"] for r in results[name]]
        summary[name] = {"ta_ms_per_round": tas, "ta_ms_median": statistics.median(tas), "ta_spread": (max(tas) - min(tas)) / statistics.median(tas),
                         "per_pass_ms_median": {k: statistics.median([r["median_ms"][k] for r in results[name]]) for k in results[name][0]["median_ms"]},
                         "per_pass_spread": {k: (max(v) - min(v)) / statistics.median(v) for k in results[name][0]["median_ms"]
                                             for v in [[r["median_ms"][k] for r in results[name]]]},
                         "sm_mhz": [r["clocks"]["sm_mhz"] for r in results[name]], "digest_mismatches": None if args.no_digest else len(mismatches[name])}
        if args.bench_steps:
            v = benches[name]
            summary[name].update({"bench_values": v, "bench_median": statistics.median(v), "bench_spread": (max(v) - min(v)) / statistics.median(v)})
            summary[name]["bench_dumps_identical_to_%s" % libs[0][0]] = all(same_files(os.path.join(dumps, "%s_%d" % (libs[0][0], r)), os.path.join(dumps, "%s_%d" % (name, r)))
                                                                           for r in range(args.rounds))
    if args.bench_steps:  # bench.py value of each build over the baseline's in the same round
        for name, _ in libs[1:]:
            summary[name]["bench_ratio_per_pair"] = [v / b0 for v, b0 in zip(benches[name], benches[libs[0][0]])]
    report["summary"] = summary
    report["mismatch_examples"] = {k: v[:10] for k, v in mismatches.items()}
    text = json.dumps(report, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(text)
    import shutil
    shutil.rmtree(dumps, ignore_errors=True)
    return 0 if all(not s["digest_mismatches"] for s in summary.values()) else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--ab", nargs="+", metavar="NAME=LIB", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--bench-steps", type=int, default=0)
    ap.add_argument("--no-digest", action="store_true", help="time the passes without copying and hashing textures between them")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.ab:
        sys.exit(driver(args))
    worker(args)


if __name__ == "__main__":
    main()
