"""GPU: parity AT the benchmark configuration (VERDICT r1 weak #3): BASELINE configs[2] - dual 128x128 cameras, batch 256 drawn
50/50 from an online ring and a demo ring (RLPD) - on the fp16 tensor-core build, through the CUDA-graph replay path that
bench.py times (1st call eager, 2nd capture + replay, 3rd replay), against the oracle on the same pre-step state.
Bars (north_star): crops / indices bit-exact, Q-values, TD targets and the loss within 1e-2 (16-bit operands)."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import fake_env, oracle_cfg_from_agent, oracle_state_from_agent, random_transitions, rel_err, to_numpy_tree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fp16_graph_replayed_step_at_b256_dual_camera_rlpd_status_clean():
    sys.path.insert(0, ROOT)
    from bench import fill_ring_synthetic
    from oracle import drq as O
    from oracle.replay import concat_batches as oconcat
    from oracle.replay import unpack
    from serl_b200.utils.launcher import make_drq_agent, make_replay_buffer
    from serl_b200.utils.train_utils import concat_batches
    torch.set_num_threads(min(os.cpu_count() or 1, 32))
    cams, B = ("cam0", "cam1"), 256
    env = fake_env(cams)
    rb = make_replay_buffer(env, capacity=3000, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=11)
    demo = make_replay_buffer(env, capacity=20 * 101, type="memory_efficient_replay_buffer", image_keys=list(cams), seed=12)
    fill_ring_synthetic(rb, seed=1)
    fill_ring_synthetic(demo, seed=2)
    tr = random_transitions(np.random.default_rng(0), 1, cams)[0]
    agent = make_drq_agent(42, tr["observations"], tr["actions"], image_keys=cams, encoder_type="resnet-pretrained", precision="fp16")
    assert agent.use_cuda_graphs
    ocfg = oracle_cfg_from_agent(agent)
    it = rb.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True})
    dit = demo.get_iterator(sample_args={"batch_size": B // 2, "pack_obs_and_next_obs": True})
    modes = []
    for step in range(3):
        ostate = oracle_state_from_agent(agent, torch.float32)
        b1, b2 = next(it), next(dit)
        both = concat_batches(b1, b2, axis=0)
        h1 = to_numpy_tree({k: v for k, v in b1.to_dict().items() if k != "_indices"})
        h2 = to_numpy_tree({k: v for k, v in b2.to_dict().items() if k != "_indices"})
        host = unpack(oconcat(h1, h2, axis=0))
        agent, info = agent.update_critics(both)
        key = agent._graph_key(("update_critics", None), both)
        modes.append("graph" if isinstance(agent._graphs.get(key), tuple) else "eager")
        oinfo = O.update_critics(ostate, ocfg, host, dtype=torch.float32)
        eng = agent._engines[B]
        for cam in cams:                                             # integer outputs: bit-exact under graph replay too
            pix = eng.pix[cam].cpu().numpy()
            np.testing.assert_array_equal(pix[:B], oinfo["_aug"]["observations"][cam][:, 0])
            np.testing.assert_array_equal(pix[B:], oinfo["_aug"]["next_observations"][cam][:, 0])
        q, tq = eng.q.cpu().numpy(), eng.target_q.cpu().numpy()
        assert np.isfinite(q).all()
        eq, et = rel_err(q, oinfo["critic"]["_q"].numpy()), rel_err(tq, oinfo["critic"]["_target_q"].numpy())
        el = abs(float(info["critic"]["critic_loss"]) - oinfo["critic"]["critic_loss"]) / max(abs(oinfo["critic"]["critic_loss"]), 1e-6)
        print(f"step {step} ({modes[-1]}): Q err {eq:.2e}, target err {et:.2e}, loss err {el:.2e}")
        assert eq < 1e-2 and et < 1e-2 and el < 1e-2, (step, eq, et, el)
        np.testing.assert_array_equal(agent.state.rng, ostate.rng)
    assert modes == ["eager", "graph", "graph"], modes
    agent.check_status()                                             # replay draws, fused heads and the trunk kernels' fault flags
