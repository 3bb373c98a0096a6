"""Byzantine attacks against each resilient aggregation rule on the C2 team: 4 cooperative agents (H = 1) and agent 4
Byzantine (include/rcmarl.h, rcmarl_attack), for every rule (by default clip, trim, wmsr; any of the coordinate rules,
the distance-based krum, mkrum, scclip, gmed, the divide-and-conquer dnc, the exact subset-selection mda and smea, and
the iterative outlier scissor ios)
x attack (alie, ipm, gauss) over the learning harness's seeds
(tests/golden/ref_learning.npz, scenario malicious/H1: the start weights and task of each seed; agent 4 keeps its weights
and learns like a Faulty agent).  Reported per cell: the cooperative team's return and the cooperative critics' estimate
of it, means of the last 500 episodes, over the seeds; for a distance-based rule, dnc, mda, smea or ios also the mean weight the receivers of
agent 4 gave its crafted message in the last epoch of the last round (Trainer.neighbour_weights, both nets), over the
seeds.  The attack list (by default alie 1.0, ipm 0.5, gauss 0.3) may also name the min-max / min-sum attacks
(rcmarl_adaptive_attack: minmax_uv, minmax_std, minmax_sgn, minsum_uv, minsum_std, minsum_sgn, scale 1 = the paper's
attack) and the rule-aware attacks tuned against each receiver's own rule and H (rcmarl_tailored_attack: tailored_uv,
tailored_std, tailored_sgn, range multiplier 2 by default); an entry is a name or name:param.  For those the table also
reports the mean gamma (gamma_i* for a tailored attack) of agent 4's messages in the last epoch of the last round
(Trainer.attack_gammas, both nets and every receiver), over the seeds.  The tailored attacks do not model dnc, mda or
smea: those cells are marked refused.  A rule may be written nnm+<rule> (e.g. nnm+mkrum): every cooperative agent then mixes the
messages it hears by nearest-neighbour mixing (rcmarl_nnm_mix) before its rule, and the weight reported for a
whole-message rule is the effective weight w M of agent 4's message.  Likewise bucket+<rule> (s = 2) or
bucket<s>+<rule> (e.g. bucket3+gmed) buckets the messages (rcmarl_bucket_mix) before the rule, which then reads the own
row and ceil(3 / s) bucket means at C2; a rule that refuses that many rows at H = 1 (krum, mkrum at s = 2) is marked
refused.  A rule may also be written m<beta>+<rule> (e.g. m0.9+scclip): every cooperative agent then keeps per-neighbour
momentum at beta (rcmarl_momentum_mix) and its rule reads the momentum rows, one per in-neighbour; the weight reported
for a whole-message rule is the weight of agent 4's momentum row.  The tailored attacks do not model mixing or momentum
either, and the pipeline-aware attacks do not model momentum: those cells are marked refused; the pipeline-aware attacks (rcmarl_pipeline_attack:
pipeline_uv, pipeline_std, pipeline_sgn, range multiplier 2 by default) model the receiver's mixing step and every rule,
dnc included, but not mda or smea, whose cells are marked refused (their gamma is reported as the tailored attacks').
The momentum-aware attacks (rcmarl_history_attack: history_uv, history_std, history_sgn, range multiplier 2 by default)
run the pipeline attack's search in a momentum receiver's momentum rows and invert its momentum step; against a
receiver without momentum they are the pipeline attacks, and mda or smea cells are marked refused.
Any of these rule names may take an arc+ prefix (e.g. arc+mkrum, arc+nnm+mkrum, arc+m0.9+scclip): every cooperative
agent then clips its k_clip = 1 furthest message (adaptive robust clipping, rcmarl_arc_clip) after its momentum step and
before its mixing step, and the weight reported for a whole-message rule is agent 4's effective weight through the
clipping factors (Trainer.neighbour_weights).  No tailored, pipeline or history attack models clipping: those cells are
marked refused.  The ARC-aware attacks (arc_uv, arc_std, arc_sgn, range multiplier 2 by default) run the history or
pipeline search through the receiver's clipping step as well (rcmarl_history_arc_attack / rcmarl_pipeline_arc_attack);
against a receiver that does not clip they are the history attacks, and mda or smea cells are marked refused.  The
subset-aware attacks (subset_uv, subset_std, subset_sgn, range multiplier 2 by default) run that search through an mda or
smea receiver's exact subset selection as well (rcmarl_subset_history_attack / rcmarl_subset_pipeline_attack); against
any other rule they are the ARC-aware attacks.  The IOS-aware attacks (ios_uv, ios_std, ios_sgn, range multiplier 2 by
default) run that search through an ios receiver's iterative outlier scissor as well (rcmarl_ios_history_attack /
rcmarl_ios_pipeline_attack); against any other rule they are the subset-aware attacks.  No other rule-aware attack
(tailored, pipeline, history, ARC-aware or subset-aware) models ios: those cells are marked refused.
The list may also name the dissensus attack (rcmarl_dissensus_attack, dissensus[:eps], eps = 1 by default: it cancels
the receiver's honest pull under a plain mean) and the mimic attack (rcmarl_mimic_attack, mimic[:T0], T0 = 50 power steps
by default, after which the direction is frozen); for mimic the table reports, per receiver, the agent whose message
agent 4 copied in the last epoch of the last round (Trainer.mimic_targets, critic / team-reward net), over the seeds.

Before the sweep it times one C2 update round at the benchmark's size with agent 4 Byzantine against the same round with
agent 4 Faulty, alternating the two trainers round by round (CUDA events around update_round).  When the rule list names
a distance-based rule it also times the round (agent 4 Byzantine) with every cooperative agent on clip, gmed and mkrum,
and when it names dnc, mda, smea or ios, on clip and each of those it names (all of them when it names several),
alternated the same way.  When the attack list names an adaptive attack it also times the round with agent 4 on
minmax_std against the same round on gauss, alternated the same way, and when it names a tailored attack, the round on
tailored_std (every cooperative agent on clip) against gauss, when it names a pipeline attack, the round on
pipeline_std against gauss, when it names a history attack, the round on history_std against gauss with every
cooperative agent on m0.9+clip, and when it names mimic, the round on mimic against gauss.

    python tools/attack_sweep.py [n_blocks=40] [n_envs=256] [timed_rounds=10] [out_dir=attack_sweep_out]
                                 [rules=clip,trim,wmsr] [attacks=alie,ipm,gauss]
        -> out_dir/attack_sweep.{json,md} (a relative out_dir is taken from the current directory)
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "resilient-consensus-based-marl_b200"))
import bench                                   # noqa: E402
import torch                                   # noqa: E402
from rcmarl._lib import RcmarlError            # noqa: E402
from rcmarl.trainer import Trainer             # noqa: E402

PARAMS = {"alie": 1.0, "ipm": 0.5, "gauss": 0.3, "tailored_uv": 2.0, "tailored_std": 2.0, "tailored_sgn": 2.0,
          "pipeline_uv": 2.0, "pipeline_std": 2.0, "pipeline_sgn": 2.0, "history_uv": 2.0, "history_std": 2.0,
          "history_sgn": 2.0, "arc_uv": 2.0, "arc_std": 2.0, "arc_sgn": 2.0,
          "subset_uv": 2.0, "subset_std": 2.0, "subset_sgn": 2.0, "ios_uv": 2.0, "ios_std": 2.0, "ios_sgn": 2.0,
          "dissensus": 1.0, "mimic": 50.0}
n_blocks = int(sys.argv[1]) if len(sys.argv) > 1 else 40
n_envs = int(sys.argv[2]) if len(sys.argv) > 2 else 256
timed_rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 10
out_dir = os.path.abspath(sys.argv[4] if len(sys.argv) > 4 else "attack_sweep_out")
RULES = tuple((sys.argv[5] if len(sys.argv) > 5 else "clip,trim,wmsr").split(","))


def split_clipping(rule):
    """(clipping, the rest) of a rule name: "arc+nnm+mkrum" -> ("arc", "nnm+mkrum"), "mkrum" -> (None, "mkrum")."""
    if rule.startswith("arc+"):
        return "arc", rule[4:]
    return None, rule


def split_momentum(rule):
    """(beta, the rest) of a rule name: "m0.9+scclip" -> (0.9, "scclip"), "scclip" -> (None, "scclip"); an arc prefix
    is dropped."""
    rule = split_clipping(rule)[1]
    if rule.startswith("m") and "+" in rule and rule[1:2].isdigit():
        beta, rest = rule[1:].split("+", 1)
        return float(beta), rest
    return None, rule


def split_rule(rule):
    """(mixing, aggregation rule) of a rule name: "nnm+mkrum" -> ("nnm", "mkrum"), "bucket+gmed" -> (("bucket", 2),
    "gmed"), "bucket3+gmed" -> (("bucket", 3), "gmed"), "mkrum" -> (None, "mkrum"); a momentum prefix is dropped."""
    rule = split_momentum(rule)[1]
    if rule.startswith("nnm+"):
        return "nnm", rule[4:]
    if rule.startswith("bucket") and "+" in rule:
        s, base = rule[6:].split("+", 1)
        return ("bucket", int(s) if s else 2), base
    return None, rule


BASES = tuple(split_rule(r)[1] for r in RULES)
VECTOR = ("krum", "mkrum", "scclip", "gmed")
SUBSET = ("mda", "smea")
WHOLE = VECTOR + ("dnc",) + SUBSET + ("ios",)   # the rules that report neighbour weights
ADAPTIVE = ("minmax_uv", "minmax_std", "minmax_sgn", "minsum_uv", "minsum_std", "minsum_sgn")
TAILORED = ("tailored_uv", "tailored_std", "tailored_sgn")
PIPELINE = ("pipeline_uv", "pipeline_std", "pipeline_sgn")
HISTORY = ("history_uv", "history_std", "history_sgn")
ARC = ("arc_uv", "arc_std", "arc_sgn")
SUBSET = ("subset_uv", "subset_std", "subset_sgn")
IOS = ("ios_uv", "ios_std", "ios_sgn")
ATTACKS = tuple((a.split(":")[0], float(a.split(":")[1]) if ":" in a else PARAMS.get(a, 1.0))
                for a in (sys.argv[6] if len(sys.argv) > 6 else "alie,ipm,gauss").split(","))
tail = 10                                       # 10 blocks x 50 episodes = the last 500 episodes


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return name, float(out.splitlines()[0])
    except Exception:
        return name, None


def timing():
    """ms per update round (median over rounds) with agent 4 Faulty and Byzantine, both at the benchmark's C2 shape."""
    cfg = bench.workload("C2", 0)
    base = dict(cfg, labels=["Cooperative"] * 4 + ["Faulty"])
    trs = {"Faulty": Trainer(**base), "Byzantine": Trainer(**dict(base, labels=["Cooperative"] * 4 + ["Byzantine"],
                                                                   attack=("gauss", 0.3)))}
    ms = {k: [] for k in trs}
    for r in range(timed_rounds + 1):
        for k, tr in trs.items():
            tr.rollout_block()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            tr.update_round()
            b.record()
            torch.cuda.synchronize()
            if r > 0:                                   # round 0 warms up
                ms[k].append(a.elapsed_time(b))
    out = {k: dict(median_ms=float(np.median(v)), rounds_ms=v) for k, v in ms.items()}
    out["added_ms"] = out["Byzantine"]["median_ms"] - out["Faulty"]["median_ms"]
    out["n_envs"] = cfg["n_envs"]
    out["attack_launches_per_round"] = trs["Byzantine"].n_epochs
    return out


def timed_rules():
    """The rules rule_timing compares: clip, then gmed and mkrum if a distance-based rule is listed, and dnc, mda,
    smea and ios where listed."""
    return (("clip",) + (("gmed", "mkrum") if any(r in VECTOR for r in BASES) else ())
            + tuple(r for r in ("dnc",) + SUBSET if r in BASES) + (("ios",) if "ios" in BASES else ()))


def rule_timing():
    """ms per update round (median over rounds) with agent 4 Byzantine (gauss) and every cooperative agent on each of
    timed_rules(), at the benchmark's C2 shape, the trainers alternated round by round."""
    cfg = dict(bench.workload("C2", 0), labels=["Cooperative"] * 4 + ["Byzantine"], attack=("gauss", 0.3))
    trs = {r: Trainer(**dict(cfg, aggregation=[r] * 4 + ["clip"])) for r in timed_rules()}
    ms = {k: [] for k in trs}
    for r in range(timed_rounds + 1):
        for k, tr in trs.items():
            tr.rollout_block()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            tr.update_round()
            b.record()
            torch.cuda.synchronize()
            if r > 0:
                ms[k].append(a.elapsed_time(b))
    out = {k: dict(median_ms=float(np.median(v)), rounds_ms=v) for k, v in ms.items()}
    for k in timed_rules()[1:]:
        out[f"{k}_added_ms"] = out[k]["median_ms"] - out["clip"]["median_ms"]
    out["n_envs"] = cfg["n_envs"]
    out["aggregation_launches_per_round"] = trs["clip"].n_epochs
    return out


def adaptive_timing(attack="minmax_std", momentum=None):
    """ms per update round (median over rounds) with agent 4 Byzantine on gauss and on `attack`, at the benchmark's C2
    shape (every cooperative agent with `momentum`), the two trainers alternated round by round."""
    cfg = dict(bench.workload("C2", 0), labels=["Cooperative"] * 4 + ["Byzantine"], momentum=momentum)
    trs = {a: Trainer(**dict(cfg, attack=(a, PARAMS.get(a, 1.0)))) for a in ("gauss", attack)}
    ms = {k: [] for k in trs}
    for r in range(timed_rounds + 1):
        for k, tr in trs.items():
            tr.rollout_block()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            tr.update_round()
            b.record()
            torch.cuda.synchronize()
            if r > 0:
                ms[k].append(a.elapsed_time(b))
    out = {k: dict(median_ms=float(np.median(v)), rounds_ms=v) for k, v in ms.items()}
    out[f"{attack}_added_ms"] = out[attack]["median_ms"] - out["gauss"]["median_ms"]
    out["n_envs"] = cfg["n_envs"]
    return out


def mean_gamma(tr):
    """Mean gamma of the adaptive, tailored, pipeline and history messages of the last epoch (critic and TR nets, every receiver)."""
    g = [x for v in tr.attack_gammas().values() for x in v.tolist()]
    return float(np.mean(g)) if g else None


def byzantine_weight(tr, b=4):
    """Mean weight the receivers of agent b gave its message in the last epoch (critic and TR nets)."""
    ws = []
    for j, w in tr.neighbour_weights().items():
        for k, node in enumerate(tr.in_nodes[j]):
            if node == b:
                ws.extend(w[:, k].tolist())
    return float(np.mean(ws)) if ws else None


z = np.load(os.path.join(ROOT, "tests", "golden", "ref_learning.npz"))
runs = [str(r) for r in z["runs"] if str(r).startswith("malicious/H1/")]
name, power = card()
result = dict(card=name, power_limit_w=power, n_blocks=n_blocks, n_envs=n_envs, timing=timing(), cells=[])
print(f"{name}, power limit {power} W: update round {result['timing']['Faulty']['median_ms']:.2f} ms (Faulty) vs "
      f"{result['timing']['Byzantine']['median_ms']:.2f} ms (Byzantine)", flush=True)
vector = any(r in WHOLE for r in BASES)


def timing_line(rt):
    return ", ".join([f"clip {rt['clip']['median_ms']:.2f} ms"] + [f"{k} {rt[k]['median_ms']:.2f} ms ({rt[k + '_added_ms']:+.3f} ms)"
                                                               for k in timed_rules()[1:]])


adaptive = any(a in ADAPTIVE + TAILORED + PIPELINE + HISTORY + ARC + SUBSET + IOS for a, _ in ATTACKS)
tailored = any(a in TAILORED for a, _ in ATTACKS)
pipeline = any(a in PIPELINE for a, _ in ATTACKS)
history = any(a in HISTORY for a, _ in ATTACKS)
mimic = any(a == "mimic" for a, _ in ATTACKS)
if vector:
    result["rule_timing"] = rt = rule_timing()
    print(f"update round with agent 4 Byzantine: {timing_line(rt)}", flush=True)
if any(a in ADAPTIVE for a, _ in ATTACKS):
    result["adaptive_timing"] = at = adaptive_timing()
    print(f"update round with agent 4 Byzantine: gauss {at['gauss']['median_ms']:.2f} ms, minmax_std "
          f"{at['minmax_std']['median_ms']:.2f} ms ({at['minmax_std_added_ms']:+.3f})", flush=True)
if tailored:
    result["tailored_timing"] = tt = adaptive_timing("tailored_std")
    print(f"update round with agent 4 Byzantine: gauss {tt['gauss']['median_ms']:.2f} ms, tailored_std "
          f"{tt['tailored_std']['median_ms']:.2f} ms ({tt['tailored_std_added_ms']:+.3f})", flush=True)
if pipeline:
    result["pipeline_timing"] = pt = adaptive_timing("pipeline_std")
    print(f"update round with agent 4 Byzantine: gauss {pt['gauss']['median_ms']:.2f} ms, pipeline_std "
          f"{pt['pipeline_std']['median_ms']:.2f} ms ({pt['pipeline_std_added_ms']:+.3f})", flush=True)
if history:
    result["history_timing"] = ht = adaptive_timing("history_std", momentum=0.9)
    print(f"update round with agent 4 Byzantine, receivers on m0.9+clip: gauss {ht['gauss']['median_ms']:.2f} ms, "
          f"history_std {ht['history_std']['median_ms']:.2f} ms ({ht['history_std_added_ms']:+.3f})", flush=True)
if mimic:
    result["mimic_timing"] = mt = adaptive_timing("mimic")
    print(f"update round with agent 4 Byzantine: gauss {mt['gauss']['median_ms']:.2f} ms, mimic "
          f"{mt['mimic']['median_ms']:.2f} ms ({mt['mimic_added_ms']:+.3f})", flush=True)


def copied_line(targets):
    """'j: critic copies / TR copies' per receiver j over the seeds, e.g. '1: 3,3,2 / 2,3,3'."""
    return "; ".join(f"{j}: " + ",".join(str(c) for c, _ in ks) + " / " + ",".join(str(t) for _, t in ks)
                     for j, ks in sorted(targets.items()))


for rule in RULES:
    for attack in ATTACKS:
        team, est, byz, gam, copied = [], [], [], [], {}
        refused = None
        for tag in runs:
            _, _, ss = tag.split("/")
            labels = [str(x) for x in z[f"{tag}/labels"]]
            assert labels == ["Cooperative"] * 4 + ["Malicious"]
            w = []
            for i in range(5):
                nets_i, n = [], 0
                while f"{tag}/agent{i}/n{n}_k0" in z.files:
                    nets_i.append([z[f"{tag}/agent{i}/n{n}_k{k}"] for k in range(6)])
                    n += 1
                w.append(nets_i[:3])
            mixing, base = split_rule(rule)
            try:
                tr = Trainer(labels=["Cooperative"] * 4 + ["Byzantine"], in_nodes=bench.IN_NODES5, weights=w,
                             desired=z[f"{tag}/desired"], n_envs=n_envs, H=1, seed=int(ss[1:]), aggregation=base,
                             attack=attack, mixing=mixing, momentum=split_momentum(rule)[0],
                             clipping=split_clipping(rule)[0], **bench.HYPER)
            except RcmarlError as ex:                   # e.g. a tailored attack against dnc, mda or mixing
                refused = str(ex)
                break
            t, e = [], []
            for _ in range(n_blocks):
                ee, rr = tr.rollout_block()
                tr.update_round()
                t.append(float(rr[:, :4].mean())); e.append(float(ee[:, :4].mean()))
            team.append(float(np.mean(t[-tail:]))); est.append(float(np.mean(e[-tail:])))
            byz.append(byzantine_weight(tr))
            gam.append(mean_gamma(tr))
            for (_, j), k in tr.mimic_targets().items():
                copied.setdefault(int(j), []).append([int(x) for x in k])
        if refused is not None:
            cell = dict(rule=rule, attack=attack[0], param=attack[1], refused=refused)
            result["cells"].append(cell)
            print(f"{rule:9s} {attack[0]:5s} {attack[1]:4.1f}: refused ({refused})", flush=True)
            continue
        cell = dict(rule=rule, attack=attack[0], param=attack[1], seeds=len(runs), team=float(np.mean(team)),
                    est=float(np.mean(est)), team_per_seed=team, est_per_seed=est)
        if vector:
            cell["byz_weight"] = float(np.mean(byz)) if split_rule(rule)[1] in WHOLE else None
        if adaptive:
            cell["gamma"] = (float(np.mean(gam)) if attack[0] in ADAPTIVE + TAILORED + PIPELINE + HISTORY + ARC + SUBSET
                             + IOS else None)
        if mimic:
            cell["copied"] = {str(j): ks for j, ks in copied.items()} if copied else None
        result["cells"].append(cell)
        print(f"{rule:9s} {attack[0]:5s} {attack[1]:4.1f}: team {cell['team']:7.2f}  estimate {cell['est']:7.2f}"
              + (f"  weight of agent 4 {cell['byz_weight']:.3f}" if cell.get("byz_weight") is not None else "")
              + (f"  gamma {cell['gamma']:.3f}" if cell.get("gamma") is not None else "")
              + (f"  copied {copied_line(copied)}" if copied else ""), flush=True)

os.makedirs(out_dir, exist_ok=True)
json.dump(result, open(os.path.join(out_dir, "attack_sweep.json"), "w"))
with open(os.path.join(out_dir, "attack_sweep.md"), "w") as f:
    f.write(f"{name}, power limit {power} W; {len(runs)} seeds, {n_blocks} blocks x 50 episodes, {n_envs} environments; "
            "means of the last 500 episodes\n\n| rule | attack | team return | critic estimate |"
            + (" weight of agent 4 |" if vector else "") + (" gamma |" if adaptive else "")
            + (" copied (receiver: critic / TR, per seed) |" if mimic else "")
            + "\n|---|---|---|---|" + ("---|" if vector else "") + ("---|" if adaptive else "") + ("---|" if mimic else "")
            + "\n")
    for c in result["cells"]:
        if "refused" in c:
            f.write(f"| {c['rule']} | {c['attack']} {c['param']} | refused | refused |" + (" - |" if vector else "")
                    + (" - |" if adaptive else "") + (" - |" if mimic else "") + "\n")
            continue
        f.write(f"| {c['rule']} | {c['attack']} {c['param']} | {c['team']:.2f} | {c['est']:.2f} |"
                + ((f" {c['byz_weight']:.3f} |" if c["byz_weight"] is not None else " - |") if vector else "")
                + ((f" {c['gamma']:.3f} |" if c["gamma"] is not None else " - |") if adaptive else "")
                + ((f" {copied_line({int(j): k for j, k in c['copied'].items()})} |" if c["copied"] else " - |")
                   if mimic else "") + "\n")
    t = result["timing"]
    f.write(f"\nC2 update round at {t['n_envs']} environments (median of {timed_rounds}, alternated): "
            f"{t['Faulty']['median_ms']:.2f} ms with agent 4 Faulty, {t['Byzantine']['median_ms']:.2f} ms Byzantine (gauss), "
            f"{t['added_ms']:+.2f} ms\n")
    if vector:
        rt = result["rule_timing"]
        f.write(f"\nC2 update round at {rt['n_envs']} environments, agent 4 Byzantine (gauss), every cooperative agent on one "
                f"rule (median of {timed_rounds}, alternated): {timing_line(rt)}\n")
    if "adaptive_timing" in result:
        at = result["adaptive_timing"]
        f.write(f"\nC2 update round at {at['n_envs']} environments, agent 4 Byzantine (median of {timed_rounds}, alternated): "
                f"gauss {at['gauss']['median_ms']:.2f} ms, minmax_std {at['minmax_std']['median_ms']:.2f} ms "
                f"({at['minmax_std_added_ms']:+.3f} ms)\n")
    if tailored:
        tt = result["tailored_timing"]
        f.write(f"\nC2 update round at {tt['n_envs']} environments, agent 4 Byzantine (median of {timed_rounds}, alternated): "
                f"gauss {tt['gauss']['median_ms']:.2f} ms, tailored_std {tt['tailored_std']['median_ms']:.2f} ms "
                f"({tt['tailored_std_added_ms']:+.3f} ms)\n")
    if pipeline:
        pt = result["pipeline_timing"]
        f.write(f"\nC2 update round at {pt['n_envs']} environments, agent 4 Byzantine (median of {timed_rounds}, alternated): "
                f"gauss {pt['gauss']['median_ms']:.2f} ms, pipeline_std {pt['pipeline_std']['median_ms']:.2f} ms "
                f"({pt['pipeline_std_added_ms']:+.3f} ms)\n")
    if history:
        ht = result["history_timing"]
        f.write(f"\nC2 update round at {ht['n_envs']} environments, agent 4 Byzantine, receivers on m0.9+clip (median "
                f"of {timed_rounds}, alternated): gauss {ht['gauss']['median_ms']:.2f} ms, history_std "
                f"{ht['history_std']['median_ms']:.2f} ms ({ht['history_std_added_ms']:+.3f} ms)\n")
    if mimic:
        mt = result["mimic_timing"]
        f.write(f"\nC2 update round at {mt['n_envs']} environments, agent 4 Byzantine (median of {timed_rounds}, alternated): "
                f"gauss {mt['gauss']['median_ms']:.2f} ms, mimic {mt['mimic']['median_ms']:.2f} ms "
                f"({mt['mimic_added_ms']:+.3f} ms)\n")
print(open(os.path.join(out_dir, "attack_sweep.md")).read())
