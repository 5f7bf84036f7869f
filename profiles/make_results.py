"""bench.py JSON lines -> a markdown results table (printed to stdout).

    python profiles/make_results.py profiles/h100_bench_second.json profiles/h100_bench_pillars.json profiles/h100_bench_cbgs.json \
        [--scale <torchrun N = 1 line> <N = 2 line> ...]
"""
import json
import sys


def load(path):
    with open(path) as fh:
        return json.loads([ln for ln in fh.read().splitlines() if ln.startswith("{")][-1])


def main():
    args = sys.argv[1:]
    scale = []
    if "--scale" in args:
        i = args.index("--scale")
        args, scale = args[:i], args[i + 1:]
    out = ["# Results (`bench.py`, synthetic clouds, CUDA-graph replay, L2 flushed between steps; GPU and power limit: "
           "profiles/README.md)", ""]
    out += ["| config | workload | clouds/s (device) | ms/step | clouds/s (e2e, host buffers) | launches/step | SM clock |",
            "|---|---|---|---|---|---|---|"]
    rows = [load(p) for p in args]
    for d in rows:
        out.append("| %s | %s | %.1f | %.3f | %.1f | %d | %s MHz |" % (
            d["config"].get("baseline_config", "?"), d["config"]["workload"], d["value"], d["ms_per_step"], d["e2e"]["value"],
            round(d["gpu_launches"] / d["steps"]), d["clocks"].get("sm_mhz")))
    out += ["", "## Rooflines (dense 3x3 and encoder: durations inside the replayed graph; the others: CUDA events around every C-ABI call of an eager pass)", ""]
    out += ["| config | kernel | bound | achieved | peak | frac | share of step |", "|---|---|---|---|---|---|---|"]
    for d in rows:
        for key in ("roofline", "roofline_encoder", "roofline_rulebook", "roofline_voxelize", "roofline_nms"):
            r = d.get(key)
            if not r:
                continue
            ach = "%.1f %s" % (r["achieved"], r["unit"]) if "achieved" in r else "%.3f ms/step" % r["kernel_ms_per_step"]
            peak = "%.1f" % r["peak"] if "peak" in r else "-"
            frac = "%.4f" % r["frac"] if "frac" in r else "-"
            share = "%.3f" % r["share_of_step"] if "share_of_step" in r else "-"
            out.append("| %s | %s | %s | %s | %s | %s | %s |" % (d["config"].get("baseline_config", "?"), r["kernel"][:90],
                                                               r["bound"], ach, peak, frac, share))
    if any(d.get("stage_ms_per_step_in_graph") for d in rows):
        out += ["", "## Stage times inside the replayed CUDA graph (external timing events at the stage boundaries) vs the eager per-call pass", "",
                "| config | stage | in graph [ms/step] | eager pass [ms/step] (adds the host cost of every call) |", "|---|---|---|---|"]
        for d in rows:
            g = d.get("stage_ms_per_step_in_graph") or {}
            e = d.get("stage_ms_per_step") or {}
            for k in g:
                out.append("| %s | %s | %.4f | %s |" % (d["config"].get("baseline_config", "?"), k, g[k], "%.4f" % e[k] if k in e else "-"))
            if g:
                out.append("| %s | **sum** | %.4f | (step: %.4f) |" % (d["config"].get("baseline_config", "?"), sum(g.values()), d["ms_per_step"]))
    out += ["", "## CPU baseline (reference path on the host cores of the same box)", ""]
    out += ["| config | port clouds/s (cores) | reference voxelizer, 1 thread: full call / loop only | pool of host cores |", "|---|---|---|---|"]
    for d in rows:
        c = d.get("cpu_baseline") or {}
        rv = c.get("reference_voxelizer") or {}
        out.append("| %s | %.2f (%s) | %s | %s |" % (
            d["config"].get("baseline_config", "?"), c.get("value", float("nan")), c.get("cores"),
            "%.1f ms / %.2f ms" % (1e3 * rv["single_thread_full_call_s"], 1e3 * rv["single_thread_loop_only_s"]) if rv.get("available") else "-",
            "%.0f clouds/s on %s workers" % (rv["pool_clouds_per_s"], rv["pool_workers"]) if rv.get("available") else "-"))
    d0 = rows[0]
    n5 = d0.get("nms_c5")
    if n5:
        ref = n5.get("reference") or {}
        out += ["", "## NMS at 100k boxes (BASELINE configs[4])", "",
                "ours %.1f ms (%d kept); reference iou3d kernel %.1f ms + D2H of the mask %.1f ms + host sweep %.1f ms = %.1f ms; "
                "keep lists equal: %s; speed-up %.1fx." % (n5["ours_ms"], n5["kept"], ref.get("kernel_ms", 0), ref.get("d2h_ms", 0),
                                                          ref.get("host_sweep_ms", 0), ref.get("total_ms", 0),
                                                          ref.get("keep_list_equal"), n5.get("speedup_vs_reference_gpu", 0))]
    if scale:
        out += ["", "## Scaling (weak: fixed clouds per GPU per step, one all-gather of the detections after the loop)", "",
                "| config | GPUs | clouds/s | ms/step | per-GPU vs N=1 |", "|---|---|---|---|---|"]
        base = {}
        for p in scale:
            d = load(p)
            key = d["config"].get("baseline_config", "?")
            if d["n_gpus"] == 1:
                base[key] = d["value"]
            eff = d["value"] / d["n_gpus"] / base[key] if key in base else float("nan")
            out.append("| %s | %d | %.1f | %.3f | %.3f |" % (key, d["n_gpus"], d["value"], d["ms_per_step"], eff))
    print("\n".join(out))


if __name__ == "__main__":
    main()
