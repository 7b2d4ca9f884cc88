"""CPU: the test-only restatement of annotate_concordance (oracle/annotate_ref.py) reproduces the reference's own output
(tests/golden/concordance_annotate.json.gz) cell by cell, raises what it raises at the same record, and gives the
cycle-skip table of the reference's unit test."""
import pytest

from oracle import annotate_ref as AR
from tests import annotate_golden as AG

EXCEPTIONS = {"ValueError": ValueError, "IndexError": IndexError, "KeyError": KeyError,
              "ZeroDivisionError": ZeroDivisionError}


@pytest.mark.parametrize("name", sorted(AG.load()["cases"]))
def test_oracle_reproduces_the_reference(name, tmp_path):
    case = AG.load()["cases"][name]
    _fa, bed = AG.write_inputs(str(tmp_path))
    got, annots = AR.annotate(AG.frame(case["input"]), AG.genome(), case["flow_order"], [bed] if case["bed"] else None)
    assert annots == case["annots"]
    AG.assert_frame_matches(got, case["output"])


@pytest.mark.parametrize("name", sorted(AG.load()["raising"]))
def test_oracle_raises_like_the_reference(name):
    case = AG.load()["raising"][name]
    df = AG.frame(case["input"])
    with pytest.raises(EXCEPTIONS[case["exception"]]):
        AR.annotate(df, AG.genome())
    # the failing row: without it the rest passes
    AR.annotate(df.drop(index=case["row"]).reset_index(drop=True), AG.genome())


def test_cycle_skip_table():
    for t in AG.load()["cycle_skip_table"]:
        assert AR.cycle_skip(t["left"], t["ref"], t["alt"], t["right"], t["flow_order"]) == t["status"], t
