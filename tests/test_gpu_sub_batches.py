"""Every search kind when the workspace budget (LGPU_WS_BYTES) cuts the batch into sub-batches of queries.

Each sub-batch re-plans on its own size, reuses the workspace of the one before it, writes an offset window of the
caller's outputs and runs its own widening pass, so a split call can take several paths at once (tensor-core shortlist
and exact kernels, filter scan and small path).  The budget is read once per process: each group of cases
(tests/sub_batch_cases.py) runs in two child processes, one with the default budget and one with a small one, and per
case this file asserts
  1. the split run equals the CPU oracle of the kind: ids, counts and distance bits;
  2. the split run equals the unsplit run, bit for bit;
  3. the split happened: the call launched more kernels under the small budget than under the default one (eager
     launches, same parameters), and where the kind has the debug entry, lgpu_debug_sub_batch_size is below the batch.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.sub_batch_cases import GROUPS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _child(group, path, budget, graphs):
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_NO_GRAPH="0" if graphs else "1", LGPU_SMALL_SLOTS="0")
    env.pop("LGPU_WS_BYTES", None)
    if budget:
        env.update(LGPU_WS_BYTES=str(budget), SUB_BATCH_ORACLE="1")
    r = subprocess.run([sys.executable, "-m", "tests.sub_batch_cases", group, str(path)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, f"{group} (LGPU_WS_BYTES={budget or 'default'}):\n{r.stdout[-2000:]}\n{r.stderr[-6000:]}"
    z = np.load(path)
    cases = {}
    for key in z.files:
        case, name = key.split("/")
        cases.setdefault(case, {})[name] = z[key]
    return cases


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """group -> (cases of the split run, cases of the unsplit run), each pair of children started once"""
    cache = {}

    def get(group):
        if group not in cache:
            budget, graphs = GROUPS[group]
            d = tmp_path_factory.mktemp(group)
            cache[group] = (_child(group, d / "split.npz", budget, graphs), _child(group, d / "whole.npz", 0, graphs))
        return cache[group]
    return get


def _bits(c, prefix=""):
    return [c[prefix + "ids"], c[prefix + "cnt"], np.asarray(c[prefix + "dist"], np.float32).view(np.uint32)]


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _report(group, split):
    sizes = {c: f"{int(v['bs'])} of {int(v['B'])}" for c, v in split.items() if "bs" in v}
    if sizes:
        print(f"\n{group}: sub-batch sizes (queries per sub-batch of the batch): {sizes}")
    print(f"{group}: launches split / whole:", {c: int(v["launches"]) for c, v in split.items() if "launches" in v})


def _check_case(group, case, s, w):
    assert _same(_bits(s), _bits(s, "o_")), f"{group}/{case}: the split run differs from the oracle"
    assert _same(_bits(s), _bits(w)), f"{group}/{case}: the split run differs from the unsplit run"
    assert int(s["launches"]) > int(w["launches"]), \
        f"{group}/{case}: {int(s['launches'])} launches under the small budget, {int(w['launches'])} under the " \
        "default: the batch was not split"
    if "bs" in s:
        assert int(s["bs"]) < int(s["B"]) and int(w["bs"]) == int(w["B"]), (group, case, int(s["bs"]), int(w["bs"]))


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_split_run_equals_the_oracle_and_the_unsplit_run(group, runs):
    split, whole = runs(group)
    _report(group, split)
    checked = 0
    for case, s in sorted(split.items()):
        if "ids" not in s:
            continue
        _check_case(group, case, s, whole[case])
        checked += 1
    assert checked >= 2, (group, sorted(split))


def test_the_tail_of_a_filter_scan_call_takes_the_small_path(runs):
    """Sub-batches of more than 1024 probe slots run the filter scan; the 11-query tail (88 slots) takes small.cu when
    LGPU_SMALL_SLOTS is left at the library's default.  How we know: the small path is 4 launches where the batched
    kernels need over 20, so the same call launches fewer kernels than with LGPU_SMALL_SLOTS=0 -- and by as much in the
    unsplit run it does not, because there no sub-batch is small."""
    split, whole = runs("pq8_small_tail")
    assert int(split["small_tail"]["launches"]) < int(split["batched_tail"]["launches"])
    assert int(whole["small_tail"]["launches"]) == int(whole["batched_tail"]["launches"])


def test_tensor_core_and_exact_coarse_steps_serve_one_call(runs):
    """With the tensor-core coarse step forced, sub-batches of 8 or more queries take it and the 5-query tail the exact
    kernels; the launch counts of the three variants differ, so the switches did select different coarse steps."""
    split, _ = runs("pq8_tc_coarse")
    for metric in ("l2", "cosine"):
        n = {v: int(split[f"{metric}_{v}"]["launches"]) for v in ("dense", "list", "exact")}
        assert len(set(n.values())) == 3, n
        assert int(split[f"{metric}_shape"]["bs"]) >= 8 and int(split[f"{metric}_shape"]["B"]) % int(split[f"{metric}_shape"]["bs"]) == 5


def test_flat_sub_batches_take_the_shortlist_and_the_tail_the_exact_kernels(runs):
    """dot always takes the exact kernels (distance matrix + select per sub-batch); an unsplit l2 call of 69 queries
    takes the tensor-core shortlist once.  The split l2 call runs 32 + 32 + 5 queries: its launches are twice the
    shortlist's plus one exact pass exactly when the two full sub-batches took the shortlist and the 5-query tail did
    not."""
    split, whole = runs("flat")
    for tag in ("", "rid_"):
        n = lambda run, c: int(run[tag + c]["launches"])
        assert n(whole, "l2_k10") > n(whole, "dot_k10")
        assert n(split, "dot_k10") == 3 * n(whole, "dot_k10")
        assert n(split, "l2_k10") == 2 * n(whole, "l2_k10") + n(whole, "dot_k10"), \
            (n(split, "l2_k10"), n(whole, "l2_k10"), n(whole, "dot_k10"))
    # 262144 rows: the filtered and the dense variant of the shortlist are different launch sequences
    split, whole = runs("flat_big")
    for run in (split, whole):
        assert int(run["filtered"]["launches"]) != int(run["dense"]["launches"])


def test_search_device_writes_only_its_window(runs):
    split, whole = runs("routes")
    for run in (split, whole):
        for tag in ("pq8_", "sq_"):
            assert bool(run[tag + "device"]["guard_clean"]), f"{tag}: rows outside [0, B * k) were written"
            # the host and the device route return the same rows
            assert _same(_bits(run[tag + "device"]), _bits(run[tag + "host"]))
            r = run[tag + "device_range"]
            assert bool(r["guard_clean"])
            cnt = r["cnt"]
            assert (cnt < 10).any()
            for b in range(len(cnt)):          # rows past `count` overwrite the caller's sentinel
                assert (r["ids"][b, cnt[b]:] == np.iinfo(np.uint64).max).all() and np.isposinf(r["dist"][b, cnt[b]:]).all()


def test_graph_replay_counts_every_sub_batch(runs):
    """warm-up and capture run eagerly (the capture's launches are counted once, by its first replay); a replay counts
    the captured launches of all sub-batches, so it matches the eager warm-up call"""
    split, whole = runs("graphs")
    for tag in ("pq8_", "sq_"):
        n = {c: int(split[tag + c]["launches"]) for c in ("warmup", "capture", "replay", "replay_other")}
        assert n["replay"] == n["warmup"] == n["replay_other"] == n["capture"], n
        assert n["replay"] > int(whole[tag + "replay"]["launches"])


def test_timeout_on_a_split_call(runs):
    split, whole = runs("timeout")
    for run in (split, whole):
        assert bool(run["impossible"]["raised"]), "a 1 ms timeout on 4001 queries did not raise TimeoutError"
        assert bool(run["impossible"]["untouched"]), "a timed-out call wrote to the caller's outputs"


def test_profiling_covers_the_whole_split_call(runs):
    """lgpu_last_filter_stats, lgpu_last_scanned_code_bytes and lgpu_last_stage_ms describe the call, not one of its
    sub-batches: the counters of the split run equal those of the unsplit run wherever they do not depend on how tiles
    interleave (queries, scanned bytes, the dense mode's flagged queries)."""
    split, whole = runs("profiling")
    B = int(split["shape"]["B"])
    rows = int(split["candidates"]["o_scanned"])
    for case in ("candidates", "cand_cap32", "dense", "exact", "ivf_binary"):
        s, w = split[case], whole[case]
        assert float(s["total_ms"]) > 0 and float(w["total_ms"]) > 0, case
        assert int(s["scanned"]) == int(w["scanned"]) > 0, (case, int(s["scanned"]), int(w["scanned"]))
        if case != "ivf_binary":
            assert int(s["scanned"]) == rows, (case, int(s["scanned"]), rows)
        filt = case in ("candidates", "cand_cap32", "dense")
        for run in (s, w):
            assert int(run["stats"][3]) == (B if filt else 0), (case, run["stats"])
    for run in (split, whole):           # 32-entry lists overflow for most queries (which ones depends on tile order)
        assert B // 2 < int(run["cand_cap32"]["stats"][2]) <= B, run["cand_cap32"]["stats"]
        assert int(run["cand_cap32"]["stats"][0]) > 0
    # the dense mode's flagged count is exact: the queries the band check cannot prove plus the ones holding a NaN
    base = int(whole["dense"]["stats"][2])
    for run in (split, whole):
        assert int(run["dense"]["stats"][2]) == base
        assert int(run["dense_3_nan"]["stats"][2]) == base + 3 and int(run["dense_3_nan"]["stats"][3]) == B
        assert int(run["dense_all_nan"]["stats"][2]) == B and int(run["dense_all_nan"]["stats"][3]) == B
