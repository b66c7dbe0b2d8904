import os, sys, json, subprocess
"""Roofline experiment for filter_groupby_tma_kernel: how much of the kernel time is the RED atomics?
SDBG_GROUPBY_DEBUG bits 1/2/4 drop the count / SUM(int) / SUM(double) RED (results are then wrong; timing only).
Needs a GPU."""
for dbg in (0, 4, 6, 7):
    env = dict(os.environ, SDBG_GROUPBY_DEBUG=str(dbg))
    out = subprocess.run([sys.executable, "bench.py", "--steps", "10", "--skip-cpu", "--skip-bm25", "--skip-e2e"], env=env, capture_output=True, text=True)
    try:
        d = json.loads(out.stdout.strip().splitlines()[-1])
        print("debug_skip", dbg, "kernel_ms", d["roofline"]["kernel_ms"], "frac", d["roofline"]["frac"], "sm_mhz", d["clocks"]["sm_mhz"], flush=True)
    except Exception as e:
        print("fail", dbg, out.stderr[-500:])
