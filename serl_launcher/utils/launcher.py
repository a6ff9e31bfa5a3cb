"""reference utils/launcher.py:50-272 -> serl_b200."""
from serl_b200.utils.launcher import (init_data_parallel, make_bc_agent, make_drq_agent, make_vice_agent, make_replay_buffer,  # noqa: F401
                                      make_sac_agent, make_trainer_config, make_wandb_logger)
