"""Dev tool: A/B of the union GEMV against a reference revision on one GPU.  Not a bench.

    python tools/gemv_union_ab.py prepare [REV]     # in a git checkout: export REV (default HEAD~1) to build/ab_parent/
    python tools/gemv_union_ab.py run OUT_DIR       # on the GPU machine, from the tree that contains build/ab_parent/

`run` records the card (nvidia-smi --query-gpu, read only), builds both trees, alternates
`bench.py --gpus 1 --steps 3 --warmup 1 --no-cpu-baseline` between them (3 runs each), reports value, e2e.value and
roofline.avg_launch_ms with their spread, the fc GEMV's rate over the UNION bytes of each wave's slices (computed here from
bench.py's seeded index stream) against the H100 SXM data-sheet 3.35 TB/s, and diffs the --dump-outputs of the two trees:
theta, grad and returns must be bit-identical, logits within the forward bound."""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARENT = os.path.join(ROOT, "build", "ab_parent")
BENCH = ["--gpus", "1", "--steps", "3", "--warmup", "1", "--no-cpu-baseline"]
HBM_GBS = 3350.0


def prepare(rev):
    os.makedirs(PARENT, exist_ok=True)
    arc = subprocess.run(["git", "-C", ROOT, "archive", rev], check=True, capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", PARENT], input=arc, check=True)
    print(f"exported {rev} to {PARENT}")


def build(tree):
    subprocess.run([sys.executable, "-c", "import __graft_entry__ as g; g.build()"], cwd=tree, check=True)


def bench(tree, dump):
    r = subprocess.run([sys.executable, "bench.py", *BENCH, "--dump-outputs", dump], cwd=tree, capture_output=True,
                       text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines or "illegal memory access" in r.stdout + r.stderr:
        raise RuntimeError(f"bench failed in {tree}:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    return json.loads(lines[-1])


def union_bytes_per_launch(steps=3, warmup=1, pop=1000, slots=256, count=250_000_000):
    """Mean over the timed waves of the bytes in the union of the fc slices [idx + off_fc, + K*N) of one wave."""
    sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]
    from dne import nets
    net = nets.make_net("LargeModel")
    P, fc = net.num_params, net.layers[3]
    K, N = fc.cin, fc.cout
    stream = np.random.RandomState(1)                    # bench.py: idx_stream
    n_pairs, per_wave = pop // 2, slots // 2
    out = []
    for gen in range(warmup + steps):
        idx = np.array([stream.randint(0, count - P + 1) for _ in range(n_pairs)], dtype=np.int64)
        if gen < warmup:
            continue
        for w0 in range(0, n_pairs, per_wave):
            s = np.sort(idx[w0:w0 + per_wave]) + fc.off_w
            total, end = 0, -1
            for a in s:
                b = a + K * N
                total += b - max(a, end) if b > end else 0
                end = max(end, b)
            out.append((4.0 * total, 4.0 * K * N * len(s)))
    u = np.array(out)
    return float(u[:, 0].mean()), float(u[:, 1].mean())


def spread(xs):
    xs = np.array(xs, dtype=float)
    return {"runs": xs.tolist(), "mean": float(xs.mean()), "min": float(xs.min()), "max": float(xs.max()),
            "spread": float(xs.max() - xs.min())}


def run(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    dumps = tempfile.mkdtemp(prefix="gemv_union_ab_")    # theta / grad dumps are large: kept out of OUT_DIR
    trees = {"parent": PARENT, "branch": ROOT}
    for t in trees.values():
        build(t)
    res = {k: [] for k in trees}
    for r in range(3):
        for name, tree in trees.items():
            res[name].append(bench(tree, os.path.join(dumps, f"{name}_{r}")))
            print(name, r, res[name][-1]["value"], flush=True)
    union, summed = union_bytes_per_launch()
    rep = {"card": card, "union_bytes_per_launch": union, "slice_bytes_per_launch": summed, "union_over_sum": union / summed}
    for name in trees:
        rs = res[name]
        rep[name] = {"value": spread([x["value"] for x in rs]),
                     "e2e_value": spread([x["e2e"]["value"] for x in rs if x.get("e2e")]),
                     "avg_launch_ms": spread([x["roofline"]["avg_launch_ms"] for x in rs]),
                     "max_abs_dlogit": [x["parity"]["max_abs_dlogit"] for x in rs if x.get("parity")]}
        ms = rep[name]["avg_launch_ms"]["mean"]
        rep[name]["gemv_gbs_over_union_bytes"] = union / (ms * 1e-3) / 1e9
        rep[name]["gemv_gbs_over_slice_bytes"] = summed / (ms * 1e-3) / 1e9
        rep[name]["frac_of_3350_over_union"] = rep[name]["gemv_gbs_over_union_bytes"] / HBM_GBS
    rep["value_gain"] = rep["branch"]["value"]["mean"] / rep["parent"]["value"]["mean"] - 1
    # outputs of the last run of each tree
    d0, d1 = os.path.join(dumps, "parent_2"), os.path.join(dumps, "branch_2")
    diff = {}
    for f in sorted(os.listdir(d0)):
        a, b = np.load(os.path.join(d0, f)), np.load(os.path.join(d1, f))
        diff[f] = {"identical": bool(np.array_equal(a, b)), "max_abs": float(np.abs(a - b).max()) if a.size else 0.0}
    rep["dump_diff"] = diff
    shutil.rmtree(dumps)
    with open(os.path.join(out_dir, "gemv_union_ab.json"), "w") as fh:
        json.dump(rep, fh, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    if sys.argv[1] == "prepare":
        prepare(sys.argv[2] if len(sys.argv) > 2 else "HEAD~1")
    else:
        run(sys.argv[2])
