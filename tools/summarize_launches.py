"""Summarise an ncu launch list (``--metrics gpu__time_duration.sum --csv``) into a markdown table.

    python tools/summarize_launches.py <launches>.csv "title" > <summary>.md
"""
import collections
import csv
import re
import sys


OURS = ("emer::", "tc::", "tcw::", "ff::", "wmn::")


def main():
    path, title = sys.argv[1], sys.argv[2]
    with open(path) as f:
        lines = [l for l in f if not l.startswith("==")]
    rows = list(csv.DictReader(lines))
    total = collections.OrderedDict()
    count = collections.Counter()
    for r in rows:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        name = re.sub(r"^void ", "", r["Kernel Name"])
        name = name.replace("at::", "").replace("emer::tc::", "tc::").replace("emer::tcw::", "tcw::")
        name = name.replace("emer::ff::", "ff::").replace("emer::wmn::", "wmn::")
        name = re.sub(r"\(.*$", "", name) if name.startswith(OURS) else name
        ns = float(r["Metric Value"].replace(",", ""))
        if r.get("Metric Unit", "ns") in ("us", "usecond"):
            ns *= 1000.0
        total[name] = total.get(name, 0.0) + ns
        count[name] += 1
    all_ns = sum(total.values())
    ours = sum(v for k, v in total.items() if k.startswith(OURS))
    print(f"# {title}\n")
    print("`ncu --metrics gpu__time_duration.sum --clock-control none` (cold-cache, serialised: compare SHARES, "
          "not absolutes).")
    print(f"{sum(count.values())} launches, {all_ns / 1e6:.2f} ms in total; library kernels (`emer::*`) "
          f"{100 * ours / all_ns:.1f} % of device time.\n")
    print("| kernel | launches | total ms | share |\n|---|---|---|---|")
    for k, v in sorted(total.items(), key=lambda kv: -kv[1])[:30]:
        print(f"| `{k[:100]}` | {count[k]} | {v / 1e6:.3f} | {100 * v / all_ns:.1f}% |")


if __name__ == "__main__":
    main()
