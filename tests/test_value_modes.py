"""The fused engine's value modes are a host-to-device contract: ``parallel/plan.py``'s ``VMODE_*`` must carry the
numbers of ``ops/csrc/plan.h``'s ``ValueMode``."""
import os
import re

from deepreduce_b200.parallel import plan

PLAN_H = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "deepreduce_b200", "ops", "csrc",
                      "plan.h")


def test_value_modes_match_plan_h():
    with open(PLAN_H) as f:
        body = re.search(r"enum ValueMode : uint32_t \{(.*?)\};", f.read(), re.S).group(1)
    device = {name.upper(): int(v) for name, v in re.findall(r"\bkVmode(\w+) = (\d+)", body)}
    host = {name[len("VMODE_"):]: v for name, v in vars(plan).items() if name.startswith("VMODE_")}
    assert device and device == host
