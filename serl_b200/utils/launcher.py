"""Launcher factories with the reference's names and hyper-parameters (utils/launcher.py:50-116,201-272):
`make_bc_agent`, `make_sac_agent`, `make_drq_agent`, `make_replay_buffer`, `make_trainer_config`, `make_wandb_logger`, and
`init_data_parallel` for a learner started under torchrun.
"""
from __future__ import annotations

import os
from typing import Optional

from ..agents.continuous.bc import BCAgent
from ..agents.continuous.drq import DrQAgent
from ..agents.continuous.sac import SACAgent
from ..data.data_parallel import SHARD_FRAMES, DataParallelDataStore, dp_rank_world
from ..data.data_store import MemoryEfficientReplayBufferDataStore, ReplayBufferDataStore


def make_bc_agent(seed, sample_obs, sample_action, image_keys=("image",), encoder_type="small", precision="fp32", device=None):
    """utils/launcher.py:26-47."""
    return BCAgent.create(
        seed, sample_obs, sample_action,
        network_kwargs={"activations": "tanh", "use_layer_norm": False, "hidden_dims": [256, 256]},
        policy_kwargs={"tanh_squash_distribution": False, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5},
        use_proprio=True, encoder_type=encoder_type, image_keys=image_keys, precision=precision, device=device)


def make_sac_agent(seed, sample_obs, sample_action, discount=0.99, device=None, **kwargs):
    """utils/launcher.py:50-76.  kwargs (e.g. critic_optimizer_kwargs, critic_network_kwargs) go to SACAgent.create_states."""
    return SACAgent.create_states(
        seed, sample_obs, sample_action,
        policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5},
        temperature_init=1e-2, discount=discount, backup_entropy=False, critic_ensemble_size=10, critic_subsample_size=2,
        device=device, **kwargs)


def make_drq_agent(seed, sample_obs, sample_action, image_keys=("image",), encoder_type="small", discount=0.96,
                   precision="fp32", device=None, **kwargs):
    """utils/launcher.py:79-116.  kwargs (e.g. critic_optimizer_kwargs, critic_network_kwargs) go to DrQAgent.create_drq."""
    return DrQAgent.create_drq(
        seed, sample_obs, sample_action, encoder_type=encoder_type, use_proprio=True, image_keys=image_keys,
        policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5},
        temperature_init=1e-2, discount=discount, backup_entropy=False, critic_ensemble_size=10, critic_subsample_size=2,
        precision=precision, device=device, **kwargs)


def make_vice_agent(seed, sample_obs, sample_action, sample_vice_obs=None, image_keys=("image",), vice_image_keys=("image",),
                    encoder_type="small", discount=0.96, precision="fp32", device=None, **kwargs):
    """utils/launcher.py:119-168.  The VICE classifier reads the agent's cameras (vice_image_keys must name the same ones) and
    its frame shapes; sample_vice_obs is accepted for the reference's signature."""
    if tuple(vice_image_keys) != tuple(image_keys):
        raise NotImplementedError(f"vice_image_keys={tuple(vice_image_keys)}: the VICE classifier reads the agent's cameras {tuple(image_keys)}")
    from ..agents.continuous.vice import VICEAgent
    return VICEAgent.create_vice(
        seed, sample_obs, sample_action, encoder_type=encoder_type, use_proprio=True, image_keys=image_keys,
        policy_kwargs={"tanh_squash_distribution": True, "std_parameterization": "exp", "std_min": 1e-5, "std_max": 5},
        vice_network_kwargs={"activations": "leaky_relu", "use_layer_norm": True, "hidden_dims": [256], "dropout_rate": 0.1},
        temperature_init=1e-2, discount=discount, backup_entropy=False, critic_ensemble_size=10, critic_subsample_size=2,
        precision=precision, device=device, **kwargs)


def make_replay_buffer(env, capacity: int = 1000000, rlds_logger_path: Optional[str] = None, type: str = "replay_buffer",
                       image_keys: list = [], preload_rlds_path: Optional[str] = None, preload_data_transform=None,
                       device=None, seed=None, data_parallel=False, priority_alpha: Optional[float] = None, priority_beta: float = 0.4, priority_eps: float = 1e-6):
    """utils/launcher.py:201-272 (RLDS logging / tfds preload are outside the hot path and unsupported).
    data_parallel=True returns the store wrapped in a `DataParallelDataStore` (collective: every rank calls it in the same
    order): a full replica per rank, fed on rank 0, with `seed` (or rank 0's drawn seed) + rank as each rank's sampler seed.
    data_parallel="shard_frames": the same store, drawing the same batches, with a frame-dedup ring's frames split over the
    ranks (each GPU holds ceil(capacity / world) + T slots of frames; data_parallel.py).
    priority_alpha (>= 0) makes the ring prioritized (proportional draws, importance weights with exponent priority_beta,
    priorities (|TD error| + priority_eps)^priority_alpha; replay_buffer.py); None keeps uniform draws.  Not combinable with
    data_parallel."""
    if priority_alpha is not None and data_parallel:
        raise NotImplementedError(f"a prioritized ring (priority_alpha) under data_parallel={data_parallel!r}: each rank would have "
                                  "to carry its written priorities to every replica")
    if rlds_logger_path or preload_rlds_path:
        raise NotImplementedError("RLDS logging / preload need oxe_envlogger + tensorflow_datasets (not on the hot path)")
    if data_parallel not in (False, True, SHARD_FRAMES):
        raise ValueError(f"data_parallel={data_parallel!r}: False, True (replicas) or {SHARD_FRAMES!r}")
    shard = data_parallel == SHARD_FRAMES
    if type == "replay_buffer":
        store = ReplayBufferDataStore(env.observation_space, env.action_space, capacity=capacity, device=device, seed=seed,
                                      priority_alpha=priority_alpha, priority_beta=priority_beta, priority_eps=priority_eps)
    elif type == "memory_efficient_replay_buffer":
        store = MemoryEfficientReplayBufferDataStore(env.observation_space, env.action_space, capacity=capacity,
                                                     image_keys=image_keys, device=device, seed=seed,
                                                     frame_shard=dp_rank_world() if shard else None, priority_alpha=priority_alpha, priority_beta=priority_beta, priority_eps=priority_eps)
    else:
        raise ValueError(f"Unsupported replay_buffer_type: {type}")
    return DataParallelDataStore(store, shard_frames=shard) if data_parallel else store


def init_data_parallel():
    """Joins the job `torchrun` started: reads RANK / WORLD_SIZE / LOCAL_RANK, makes cuda:LOCAL_RANK the current device and,
    with more than one rank, initialises the NCCL default process group (once; later calls only return).  Without torchrun's
    variables this is a single process on cuda:0.  Returns (rank, world)."""
    import torch
    import torch.distributed as dist
    local, world = int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(local)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", rank=int(os.environ["RANK"]), world_size=world, device_id=torch.device("cuda", local))
    if dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def make_trainer_config(port_number: int = 5488, broadcast_port: int = 5489):
    """utils/launcher.py:171-177 (needs agentlace, which is consumed unchanged)."""
    from agentlace.trainer import TrainerConfig
    return TrainerConfig(port_number=port_number, broadcast_port=broadcast_port, request_types=["send-stats"])


def make_wandb_logger(project: str = "agentlace", description: str = "serl_launcher", debug: bool = False):
    """utils/launcher.py:180-198."""
    from ..common.wandb import WandBLogger
    cfg = WandBLogger.get_default_config()
    cfg.update({"project": project, "exp_descriptor": description, "tag": description})
    return WandBLogger(wandb_config=cfg, variant={}, debug=debug)
