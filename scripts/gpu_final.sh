# End-of-round verification on one GPU: smoke, GPU parity tests, DRAM traffic (ncu) for the roofline.traffic fields,
# launch list of the default command, the default bench line (all legs) and the reference arm.
mkdir -p gpurun_out
timeout 600 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/f_smoke.log 2>&1; echo "smoke exit $?" >> gpurun_out/f_smoke.log
timeout 1500 python -m pytest tests -m gpu -q > gpurun_out/f_pytest.log 2>&1; echo "pytest exit $?" >> gpurun_out/f_pytest.log
K='ldb_(inflate_decode_kernel|inflate_resolve_kernel|deflate_lz_kernel)'
timeout 900 ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none -k regex:"$K" -s 3 -c 6 --csv --log-file gpurun_out/f_traffic_rt.csv python bench.py --steps 1 --warmup 3 --no-e2e --no-cpu --no-extra > gpurun_out/f_traffic_rt.log 2>&1
python scripts/ncu_traffic.py gpurun_out/f_traffic_rt.csv roundtrip_L6_65536x65536 > gpurun_out/f_traffic_rt.json 2>&1
timeout 900 ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none -k regex:"$K" -s 2 -c 4 --csv --log-file gpurun_out/f_traffic_dec.csv python bench.py --workload decompress --steps 1 --warmup 3 --no-e2e --no-cpu > gpurun_out/f_traffic_dec.log 2>&1
python scripts/ncu_traffic.py gpurun_out/f_traffic_dec.csv decompress_L6_65536x65536 > gpurun_out/f_traffic_dec.json 2>&1
cp profiles/dram_traffic.json gpurun_out/f_dram_traffic.json
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 60 --csv --log-file gpurun_out/f_launches.csv python bench.py --steps 2 --warmup 3 --no-e2e --no-cpu --no-extra > gpurun_out/f_launches.log 2>&1
timeout 600 python bench.py --impl reference --steps 3 --warmup 3 > gpurun_out/f_bench_ref.json 2> gpurun_out/f_bench_ref.err
timeout 900 python bench.py > gpurun_out/f_bench.json 2> gpurun_out/f_bench.err; echo "exit $?" >> gpurun_out/f_bench.err
timeout 600 python bench.py --workload decompress --steps 10 --warmup 3 > gpurun_out/f_bench_dec.json 2> gpurun_out/f_bench_dec.err; echo "exit $?" >> gpurun_out/f_bench_dec.err
tail -2 gpurun_out/f_smoke.log; tail -3 gpurun_out/f_pytest.log; cat gpurun_out/f_traffic_rt.json gpurun_out/f_traffic_dec.json
python - <<'PY'
import json
for f in ("f_bench_ref", "f_bench", "f_bench_dec"):
    try:
        d = json.loads([l for l in open("gpurun_out/%s.json" % f) if l.startswith("{")][-1])
        print(f, {k: d.get(k) for k in ("impl", "value", "ms_per_step", "ratio", "kernel_ms_per_step")}, "roofline", d.get("roofline") and {k: d["roofline"].get(k) for k in ("kernel", "achieved", "frac", "traffic_over_algorithmic")},
              "north", d.get("roofline_inflate") and {k: d["roofline_inflate"].get(k) for k in ("achieved", "frac", "traffic_over_algorithmic")},
              "e2e", d.get("e2e") and d["e2e"]["value"], "cpu", d.get("cpu_baseline") and {k: d["cpu_baseline"].get(k) for k in ("value", "cores", "per_thread_MBps")}, "clocks", d.get("clocks"))
    except Exception as e:
        print(f, "ERR", e)
PY
