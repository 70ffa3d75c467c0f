"""`python -m parallax_b200.tools.launch_ps` — the parameter-server *placement planner*.

The reference's `parallax/core/python/tools/launch_ps.py:22-53` starts one
`tf.train.Server(job_name='ps')` per host and joins it; which variable lives on which
server is decided by `GreedyLoadBalancingStrategy` (`ps/between_graph_parallel.py:49-70`).
On an NVSwitch box there is nothing to start — the server of a variable is the GPU that
owns it, served by that GPU's worker process — but the placement decision is the same
one, and this tool answers it offline with exactly the code the engine runs
(`parallel.layout.assign_owners`):

    # owner map of the sparse variables of an exported analysis, on 8 owners
    python -m parallax_b200.tools.launch_ps --analysis out/analysis_worker_0.json --owners 8
    # or variables given by hand: name:rows:dim[:partitions[:slots]]; '+' joins a
    # co-lookup group; `slots` is a count of D-wide fp32 slots or an optimizer kind
    # (`rowwise_adagrad` keeps one fp32 per row)
    python -m parallax_b200.tools.launch_ps --owners 8 \
        emb:793470:512:32:1 softmax_w:793470:512:32:1+softmax_b:793470:1:32:1
    python -m parallax_b200.tools.launch_ps --owners 8 emb:793470:512:32:rowwise_adagrad

It prints, per owner, the partitions and bytes it would hold, the imbalance of the
byte-greedy placement and of naive round-robin (`PSConfig.boundary_among_servers=False`),
and exits non-zero when a table cannot be placed (partition counts of a group differ).
The reference's flags (`--ps_hosts --worker_hosts --job_name --task_index --protocol`) are
accepted: `--worker_hosts` sets the owner count.
"""
import argparse
import json
import sys

from .. import optim
from ..parallel.layout import assign_owners


def _parse_var(spec):
    f = spec.split(":")
    if len(f) < 3:
        raise ValueError("variable spec %r: want name:rows:dim[:partitions[:slots]]" % spec)
    slots = f[4] if len(f) > 4 else 0
    if isinstance(slots, str) and not slots.isdigit():
        if slots not in optim.NUM_SLOTS:
            raise ValueError("variable spec %r: slots %r is neither a count nor an optimizer "
                             "kind (%s)" % (spec, slots, ", ".join(optim.NUM_SLOTS)))
    else:
        slots = int(slots)
    return {"name": f[0], "rows": int(f[1]), "dim": int(f[2]),
            "partitions": int(f[3]) if len(f) > 3 else None, "slots": slots}


def row_bytes(v):
    """Owner bytes of one row of variable `v`: the padded fp32 row and its slots, `slots`
    D-wide slots or those of the optimizer kind it names."""
    if isinstance(v["slots"], str):
        return optim.table_row_bytes(v["slots"], v["dim"])
    return ((v["dim"] + 3) // 4 * 16) * (1 + v["slots"])


def plan(groups, owners, greedy=True):
    """groups: list of lists of variable dicts.  Returns (owner map per group key, bytes per
    owner)."""
    items = []
    for gi, grp in enumerate(groups):
        parts = {v["partitions"] or owners for v in grp}
        if len(parts) != 1:
            raise ValueError("group %s: members differ in partition count %s"
                             % ([v["name"] for v in grp], sorted(parts)))
        P = parts.pop()
        nbytes = sum(((v["rows"] + P - 1) // P) * row_bytes(v) for v in grp)
        items.append((gi, P, nbytes))
    placed = assign_owners(items, owners) if greedy else \
        {gi: [p % owners for p in range(P)] for gi, P, _ in items}
    load = [0] * owners
    for gi, P, nbytes in items:
        for o in placed[gi]:
            load[o] += nbytes
    return placed, load


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("variables", nargs="*", help="name:rows:dim[:partitions[:slots]], "
                                                 "'+' joins a co-lookup group")
    ap.add_argument("--analysis", help="analysis_worker_*.json written by "
                                       "Config(export_graph_path=...)")
    ap.add_argument("--owners", type=int, default=None)
    ap.add_argument("--ps_hosts", default="")
    ap.add_argument("--worker_hosts", default="")
    ap.add_argument("--job_name", default="ps")
    ap.add_argument("--task_index", type=int, default=0)
    ap.add_argument("--protocol", default="grpc")
    a = ap.parse_args(argv)
    owners = a.owners or len([h for h in a.worker_hosts.split(",") if h]) or 1
    groups = [[_parse_var(v) for v in spec.split("+")] for spec in a.variables]
    if a.analysis:
        with open(a.analysis) as f:
            rep = json.load(f)
        for name, t in sorted(rep.get("tables", {}).items()):
            groups.append([{"name": name, "rows": t["V"], "dim": t["D"],
                            "partitions": t["P"], "slots": 0}])
    if not groups:
        ap.error("no variables: pass specs or --analysis")
    try:
        placed, load = plan(groups, owners, greedy=True)
        _, load_rr = plan(groups, owners, greedy=False)
    except ValueError as e:
        print("error: %s" % e, file=sys.stderr)
        return 2
    print("%d owner GPU(s); sparse variables are served over NVLink peer memory "
          "(requested protocol: %s)" % (owners, a.protocol))
    for gi, grp in enumerate(groups):
        print("  %-40s P=%-4d owners of partitions: %s"
              % ("+".join(v["name"] for v in grp), len(placed[gi]), placed[gi]))
    mean = sum(load) / float(owners)
    for o in range(owners):
        print("  owner %d: %.1f MiB" % (o, load[o] / 2 ** 20))
    imb = lambda l: (max(l) / mean - 1.0) * 100 if mean else 0.0
    print("imbalance (max over mean): byte-greedy %.1f %%, round-robin %.1f %%"
          % (imb(load), imb(load_rr)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
