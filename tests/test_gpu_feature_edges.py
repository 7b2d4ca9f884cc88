"""GPU: the feature edge corpus (tests/feature_cases.py) through both K1 tiers (the k1_tok tile kernel and the generic
parser, UGVC_K1_LEGACY=1) and both K3 paths (features assembled inside k3_heap's tile load, or K2 + k3_infer), for
the single_sample, deep_variant, deep_variant_extended and CNV plans under LR, sklearn GB of depth 8 and 10 and an
xgboost JSON document.

* The raw slot words are the same in both tiers, and the features equal the reference transformer's bit for bit.
* Each tier is used as intended: only the records the corpus marks (strings over 31 bytes, region values) are handed
  to the generic parser.
* The fused check: ``filter_batch(text)`` and ``predict_features(reference matrix)`` run the same K3 instantiation on
  the same loaded plan, one on K1's raw slots and one on the dense matrix.  Their FILTER, probabilities, qual and fp64
  likelihoods must be bit-identical, so the features K3 scores are the reference's.
* Refusals: a case the reference raises on, put at record r of a clean batch, is refused naming record r, with the
  same (record, column, reason) in both tiers and both K3 paths; with a second bad record later, r is still named."""
import os
from functools import lru_cache

import numpy as np
import pytest

from oracle import xgb_predictor as XP
from tests import feature_cases as FC
from tests import util
from variantcalling_b200 import lib
from variantcalling_b200 import model_compiler as MC
from variantcalling_b200.vcf_header import VcfHeader

pytestmark = pytest.mark.gpu

N_CLEAN = 120
AT, LATER = 17, 31


@lru_cache(maxsize=None)
def fitted(name):
    fl = FC.flavour(name)
    tr, x, _ = FC.reference_matrix(fl, fl["lines"])
    return fl, tr, x


@lru_cache(maxsize=None)
def plan_of(name, kind):
    from sklearn.ensemble import GradientBoostingClassifier

    fl, tr, x = fitted(name)
    y = fl["labels"]
    if kind == "lr":
        model = util.fit_model("lr", x, y)
    elif kind == "xgb":
        model = XP.sklearn_gb_to_xgb_json(util.fit_model("gb_small", x, y))
    else:
        depth = {"gb8": 8, "gb10": 10}[kind]
        model = GradientBoostingClassifier(n_estimators=12, learning_rate=0.2, max_depth=depth, min_samples_leaf=1,
                                           random_state=0).fit(x, y)
    return MC.compile_plan(VcfHeader("\n".join(fl["header"]) + "\n"), tr, model, fl["customs"])


def run(ctx, blob, lines, learn, legacy, phreds=False):
    text = ("\n".join(lines) + "\n").encode()
    if legacy:
        os.environ["UGVC_K1_LEGACY"] = "1"
    try:
        ctx.load_plan(blob)
        ctx.enable_phreds(2 if phreds else 0)
        ctx.reserve(len(text) + 4096, len(lines) + 16, 1)
        ctx.set_key_order(*lib.learn_key_order(learn))
        try:
            out = ctx.filter_batch(text)
        except lib.UgvcDataError:
            return {"error": ctx.last_data_error()}
        n = out["n_records"]
        res = dict(n=n, raw=ctx.debug_raw(n).copy(), low=out["low_score"].copy(), probs=out["probs"].copy(),
                   qual=out["qual"].copy(), slow=ctx.slow_records(0))
        if phreds:
            res["p64"] = ctx.collect_phreds(0, n)
        res["feats"] = ctx.debug_features(n).T.copy()
        return res
    finally:
        os.environ.pop("UGVC_K1_LEGACY", None)


def ok_cases(name):
    return [c for c in FC.cases_of(name) if c.want != FC.RAISES and c.on_device != FC.RAISES]


def bad_cases(name):
    return [c for c in FC.cases_of(name) if c.on_device == FC.RAISES]


KINDS = ["lr", "gb8", "gb10", "xgb"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", FC.FLAVOURS)
def test_features_tiers_and_fused_scores(gpu_ctx, name, kind):
    fl, tr, _ = fitted(name)
    plan = plan_of(name, kind)
    base = FC.base_record(fl)
    cases = ok_cases(name)
    clean = fl["lines"][:N_CLEAN]
    lines = clean + [FC.apply(base, c.edits) for c in cases]
    learn = ("\n".join(clean) + "\n").encode()
    _, _, want = FC.reference_matrix(fl, lines, tr)
    # each tier used as intended: the clean records' hand-overs plus the cases marked slow
    # (where even the clean base record is handed over, as in the DeepVariant and CNV sets, every case is)
    base_slow = run(gpu_ctx, plan.blob, [base], learn, legacy=False)["slow"]
    handed = run(gpu_ctx, plan.blob, clean, learn, legacy=False)["slow"] + sum(c.slow or base_slow for c in cases)
    slow = run(gpu_ctx, plan.blob, lines, learn, legacy=True)
    fast = run(gpu_ctx, plan.blob, lines, learn, legacy=False, phreds=True)
    for res, tier in ((fast, "tile"), (slow, "generic")):
        assert "error" not in res, (tier, res.get("error"), lines[res["error"][0]] if "error" in res else None)
        bad = np.argwhere(res["feats"].view(np.uint32) != want.view(np.uint32))
        if bad.size:
            r, f = bad[0]
            who = cases[r - N_CLEAN].name if r >= N_CLEAN else f"clean record {r}"
            pytest.fail(f"[{tier}] {len(bad)} features differ, first {who} / {plan.feature_names[f]}: "
                        f"{res['feats'][r, f]!r} vs {want[r, f]!r}")
    diff = np.argwhere(fast["raw"] != slow["raw"])
    assert diff.size == 0, f"slot words differ between the tiers at (slot, record) {diff[0]}"
    assert fast["slow"] == handed, (fast["slow"], handed)
    # the fused check, on the plan and reservation the tile run left: the same K3 instantiation on the reference matrix
    dense = gpu_ctx.predict_features(want)
    p64 = gpu_ctx.collect_phreds(0, len(lines))
    assert np.array_equal(fast["low"], dense["low_score"])
    assert fast["probs"].tobytes() == dense["probs"].tobytes()
    assert fast["qual"].tobytes() == dense["qual"].tobytes()
    assert fast["p64"].tobytes() == p64.tobytes()


def test_k3_paths_are_the_ones_named(gpu_ctx):
    for kind, kernel in (("gb8", "heap"), ("gb10", "infer")):
        gpu_ctx.load_plan(plan_of("ss", kind).blob)
        assert gpu_ctx.k3_config()["kernel"].startswith(kernel), (kind, gpu_ctx.k3_config())


@pytest.mark.parametrize("name", FC.FLAVOURS)
def test_refusals_name_the_record_in_both_tiers_and_both_k3_paths(gpu_ctx, name):
    fl, tr, _ = fitted(name)
    base = FC.base_record(fl)
    clean = fl["lines"][:40]
    learn = ("\n".join(fl["lines"][:N_CLEAN]) + "\n").encode()
    FC.reference_matrix(fl, clean, tr)
    other = next(c for c in bad_cases(name) if c.want == FC.RAISES)
    got = {}
    for kind in ("gb8", "gb10"):
        blob = plan_of(name, kind).blob
        for legacy in (False, True):
            for c in bad_cases(name):
                one = list(clean)
                one[AT] = FC.apply(base, c.edits)
                two = list(one)
                two[LATER] = FC.apply(base, other.edits)
                for what, lines in (("one", one), ("two", two)):
                    res = run(gpu_ctx, blob, lines, learn, legacy)
                    assert "error" in res, (c.name, kind, legacy, what)
                    got.setdefault((c.name, what), {})[(kind, legacy)] = res["error"]
    for c in bad_cases(name):
        if c.want == FC.RAISES:
            with pytest.raises((ValueError, KeyError, AssertionError, TypeError, IndexError)):
                FC.reference_matrix(fl, clean[:AT] + [FC.apply(base, c.edits)] + clean[AT + 1:], tr)
        for what in ("one", "two"):
            errs = got[(c.name, what)]
            assert len(set(errs.values())) == 1, (c.name, what, errs)
            rec, _col, reason = next(iter(errs.values()))
            assert rec == AT and reason != 0, (c.name, what, errs)

