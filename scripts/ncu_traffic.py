"""Parses `ncu --csv --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum` output of a
bench.py run and records DRAM bytes per launch of the hot kernels in profiles/dram_traffic.json, keyed by
the bench configuration.  bench.py fills roofline.traffic from that file when the configuration matches."""
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    log, key = sys.argv[1], sys.argv[2]
    rows = [r for r in csv.reader(open(log, errors="replace")) if len(r) > 5]
    hdr = next(r for r in rows if "Kernel Name" in r)
    ik, im, iv, iu = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    iid = hdr.index("ID")
    per = {}
    for r in rows:
        if r is hdr or len(r) <= iv or r[ik] == "Kernel Name":
            continue
        name = r[ik].split("(")[0]
        if not name.startswith(("ldb_inflate_decode_kernel", "ldb_inflate_resolve_kernel", "ldb_deflate_lz_kernel")):
            continue
        val = float(r[iv].replace(",", ""))
        unit = r[iu].lower()
        scale = {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9, "tbyte": 1e12}.get(unit, 1)
        per.setdefault((name, r[iid]), {})[r[im]] = val * scale
    out = {}
    for (name, _), m in per.items():
        if "dram__bytes_read.sum" in m and "dram__bytes_write.sum" in m:
            out.setdefault(name, []).append(m["dram__bytes_read.sum"] + m["dram__bytes_write.sum"])
    path = os.path.join(ROOT, "profiles", "dram_traffic.json")
    db = json.load(open(path)) if os.path.exists(path) else {}
    db[key] = {k: {"dram_bytes_per_launch": sum(v) / len(v), "launches_measured": len(v)} for k, v in out.items()}
    db[key]["source"] = "ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum (scripts/ncu_traffic.py)"
    os.makedirs(os.path.dirname(path), exist_ok=True)
    json.dump(db, open(path, "w"), indent=1, sort_keys=True)
    print(json.dumps(db[key]))


if __name__ == "__main__":
    main()
