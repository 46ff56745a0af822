"""CPU tests of host-side rules added in round 2 (no device needed)."""
import os

import pytest


def test_ulysses_subgroup_rule_keeps_twelve_waves_per_launch():
    """Head sub-groups are used only while each sub-group's attention launch keeps >= 12 waves of CTAs on
    132 SMs x 1 CTA (jenga_b200/ulysses.py); an explicit request must divide the heads."""
    from jenga_b200.ulysses import UlyssesFusedAttention as U
    n = U._n_groups
    assert n(12, None, 902) == 3          # N=2 at HY-720p: 4 heads x 902 q blocks = 27.3 waves per launch
    assert n(3, None, 902) == 1           # N=8: one head per launch would be 6.8 waves
    assert n(6, None, 902) == 3           # N=4: 2 x 902 = 13.7 waves per launch (3 groups)
    assert n(6, None, 600) == 2           # 2 x 600 = 9.1 waves (3 groups) is too few, 3 x 600 = 13.6 (2 groups)
    assert n(6, None, 400) == 1           # 6.1 waves (3 groups), 9.1 (2 groups): neither reaches 12
    assert n(12, None, None) == 3         # no shape given: the head count decides
    assert n(12, 2, 902) == 2 and n(12, 1, 902) == 1
    with pytest.raises(ValueError):
        n(12, 5, 902)


def test_fp8_pv_is_opt_in():
    """The FP8 P.V variant is never on by default (lower precision than the reference)."""
    import subprocess
    import sys
    env = {k: v for k, v in os.environ.items() if k != "JENGA_PV_FP8"}
    out = subprocess.run([sys.executable, "-c", "import jenga_b200.attention as A; print(A.PV_FP8)"],
                         capture_output=True, text=True, env=env, check=True).stdout.strip()
    assert out == "False"


def test_integration_doc_lists_every_environment_switch():
    """INTEGRATION.md's table of switches covers every JENGA_* variable the library reads."""
    import re
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    used = set()
    for f in list((root / "jenga_b200").glob("*.py")) + list((root / "jenga_b200" / "csrc").glob("*.cu")) + [root / "bench.py"]:
        used |= set(re.findall(r'(?:getenv\(|environ(?:\.get\(|\[))"(JENGA_[A-Z0-9_]+)"', f.read_text()))
    doc = (root / "INTEGRATION.md").read_text()
    missing = sorted(v for v in used if v not in doc)
    assert not missing, missing
