"""reference agents/continuous/vice.py -> serl_b200."""
from serl_b200.agents.continuous.vice import VICEAgent  # noqa: F401
