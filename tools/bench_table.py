#!/usr/bin/env python3
"""Markdown tables from bench.py JSON lines.
usage: python tools/bench_table.py bench_n1.json [bench_reference_arm.json] [more GPU-arm lines ...]"""
import json
import sys


def load(p):
    return json.loads(open(p).read().strip().splitlines()[-1])


gpu = [load(p) for p in sys.argv[1:]]
ref = [d for d in gpu if d.get("impl") == "reference"]
gpu = [d for d in gpu if d.get("impl") != "reference"]
for d in gpu:
    n = d["n_gpus"]
    print(f"### {n} GPU(s)  (steps {d['steps']}, warm-up {d['warmup']}, SM clock {d['clocks']['sm_mhz']} MHz, throttle reasons {d['clocks']['reasons']})\n")
    print("| config | kernel plan | ms / batch | instances/s | ADMM it/s/GPU | solved | mean it | algorithmic GB/s (frac of HBM peak) | e2e ms (inst/s) | reference CPU inst/s (threads, 1-thread) | GPU/CPU |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    cb = d.get("cpu_baseline") or {}
    rows = [("C2 (headline)", d.get("plan") or d["config"], d["ms_per_step"], d["value"], d["admm_iters_per_s_per_gpu"], d["solved_fraction"], 100.0, d["roofline"], d["e2e"], cb)]
    for k, v in (d.get("configs") or {}).items():
        rows.append((k, v["plan"], v["ms_per_step"], v["value"], v["admm_iters_per_s_per_gpu"], v["solved_fraction"], v["mean_iters"], v["roofline"], v.get("e2e"),
                     v.get("cpu_reference") or {}))
    for name, plan, ms, val, its, sol, mi, roof, e2e, c in rows:
        pl = f"{plan['kernel']} L={plan['lanes_per_instance']} {plan['instances_per_cta']}/SM"
        e = f"{e2e['ms_per_step']:.2f} ({e2e['value']:.3e})" if e2e else "—"
        cpu = f"{c['value']:.0f} ({c['cores']}, {c['one_thread']:.0f})" if c.get("value") else "—"
        ratio = f"{val / c['value'] / n:.0f}x" if c.get("value") else "—"
        print(f"| {name} | {pl} | {ms:.3f} | {val:.3e} | {its:.3e} | {sol:.2f} | {mi:.1f} | {roof['achieved']:.1f} ({roof['frac']:.5f}) | {e} | {cpu} | {ratio} |")
    print()
for r in ref:
    c = r["cpu_baseline"]
    print(f"### reference arm (`--impl reference`): {r['value']:.0f} instances/s on {c['cores']} threads (host: {c['host']}), 1 thread {c['one_thread']:.0f}, per core {c['per_core']:.0f}, parallel speed-up {c['parallel_speedup']:.1f}\n")
    print("| config | instances/s | threads | 1-thread | per core | mean it |")
    print("|---|---|---|---|---|---|")
    print(f"| C2 | {r['value']:.0f} | {c['cores']} | {c['one_thread']:.0f} | {c['per_core']:.0f} | {c['mean_iters']:.1f} |")
    for k, v in (r.get("configs") or {}).items():
        cc = v.get("cpu_reference")
        if cc:
            print(f"| {k} | {cc['value']:.0f} | {cc['cores']} | {cc['one_thread']:.0f} | {cc['per_core']:.0f} | {cc['mean_iters']:.1f} |")
