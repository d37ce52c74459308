# Last check of the round on one GPU: smoke, the whole GPU suite, the default bench line (no profiler runs)
mkdir -p gpurun_out
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/z_smoke.log 2>&1; echo "smoke exit $?" >> gpurun_out/z_smoke.log
timeout 900 python -m pytest tests -m gpu -q > gpurun_out/z_pytest.log 2>&1; echo "pytest exit $?" >> gpurun_out/z_pytest.log
timeout 600 python bench.py --no-l12 > gpurun_out/z_bench.json 2> gpurun_out/z_bench.err; echo "exit $?" >> gpurun_out/z_bench.err
tail -2 gpurun_out/z_smoke.log; tail -3 gpurun_out/z_pytest.log
python - <<'PY'
import json
d = json.loads([l for l in open("gpurun_out/z_bench.json") if l.startswith("{")][-1])
print({k: d.get(k) for k in ("value", "ms_per_step", "ratio", "kernel_ms_per_step")}, "e2e", d["e2e"]["value"], "north", d["roofline_inflate"]["frac"], d["extra"]["decompress_reference_streams"]["ms_per_step"], d["clocks"])
PY
