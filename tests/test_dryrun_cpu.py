"""CPU: walks the whole Python orchestration (replay ring bookkeeping, batch handles, agent update paths, launch
counting) with the kernel launches replaced by a recorder.  No arithmetic is checked here (that is the GPU
suite's job); this pins the host logic: which C-ABI entry points a step calls, in which order, and that the
host ring bookkeeping equals the reference semantics (via the oracle ring)."""
import types

import numpy as np
import pytest
import torch

from helpers import fake_env, random_transitions


@pytest.fixture()
def dry(monkeypatch):
    from serl_b200 import _lib as L
    calls = []
    real_call = L.call

    def fake_call(name, *args):
        if name.startswith("serl_host_"):
            return real_call(name, *args)
        calls.append(name)
        return 0

    class Ev:
        def record(self): pass
        def synchronize(self): pass
        def make_current_stream_wait(self): pass

    monkeypatch.setattr(L, "call", fake_call)
    monkeypatch.setattr(L, "require_cuda", lambda d: None)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    monkeypatch.setattr(L, "new_event", lambda: Ev())
    monkeypatch.setattr(L, "pin", lambda t: t)
    monkeypatch.setattr(L, "launch_count", lambda: len(calls))
    return calls


def _ring(cams, cap, hw=16, T=1):
    from serl_b200.utils.launcher import make_replay_buffer
    return make_replay_buffer(fake_env(cams, hw, T), capacity=cap, type="memory_efficient_replay_buffer", image_keys=list(cams),
                              device="cpu", seed=5)


@pytest.mark.parametrize("T,cap,n", [(1, 37, 150), (2, 23, 120)])
def test_host_ring_bookkeeping_equals_reference_semantics(dry, T, cap, n):
    from oracle.replay import OracleFrameRing
    cams = ("a", "b")
    rb = _ring(cams, cap, 8, T)
    ora = OracleFrameRing(cap, cams, (8, 8, 3), T, 7, 4)
    for tr in random_transitions(np.random.default_rng(T), n, cams, 8, T, mean_ep=6):
        rb.insert(tr)
        ora.insert(tr)
        assert len(rb) == ora.size and rb._insert_index == ora.cursor and rb._first == ora.episode_start
        np.testing.assert_array_equal(rb._valid_host, ora.valid)
    rb.flush()
    assert "serl_replay_scatter" in dry and "serl_replay_commit" in dry


def test_staging_records_are_what_the_scatter_kernel_will_read(dry):
    """Host insert path: every staged slot write is one interleaved record; field k of row r must sit at
    header + r*row_bytes + offset(k) - the addressing serl_replay_scatter uses with row_stride = row_bytes."""
    cams = ("a", "b")
    rb = _ring(cams, 50, 8, 1)
    trs = random_transitions(np.random.default_rng(3), 5, cams, 8, 1, mean_ep=100)
    for tr in trs:
        rb.insert(tr)
    n = rb._n_pending
    assert n >= len(trs)                                     # frame-dedup inserts stage obs and next_obs slots
    raw = rb._stage_host[rb._cur].numpy()
    st = rb._stn[rb._cur]
    hb, rbytes, f = rb._hdr_bytes, rb._row_bytes, rb._fields
    assert rbytes % 16 == 0 and hb % 16 == 0
    for k in range(n):
        base = hb + k * rbytes
        for c in cams:
            off, _, shape = f[("frames", c)]
            np.testing.assert_array_equal(raw[base + off: base + off + int(np.prod(shape))].reshape(shape), st["frames"][c][k])
        for name in ("state", "next_state", "actions", "rewards", "masks"):
            off, _, shape = f[name]
            np.testing.assert_array_equal(raw[base + off: base + off + 4 * shape[0]].view(np.float32), np.atleast_1d(st[name][k]))
        for name in ("dst", "src"):
            assert raw[base + f[name][0]: base + f[name][0] + 4].view(np.int32)[0] == st[name][k]
        for name in ("dones", "valid"):
            assert raw[base + f[name][0]] == st[name][k]
    # the staged frames are the inserted ones (last transition's next observation went to the last record)
    np.testing.assert_array_equal(st["frames"]["a"][n - 1], np.asarray(trs[-1]["next_observations"]["a"]).reshape(8, 8, 3))
    cur = rb._cur
    rb.flush()
    assert rb._cur == cur ^ 1 and rb._n_pending == 0          # double-buffered: the next inserts go to the other buffer


def test_drq_learner_iteration_call_sequence(dry):
    from serl_b200.utils.launcher import make_drq_agent
    from serl_b200.utils.train_utils import concat_batches
    cams = ("front", "wrist")
    rb, demo = _ring(cams, 64, 128), _ring(cams, 32, 128)
    trs = random_transitions(np.random.default_rng(0), 40, cams, 128)
    for tr in trs:
        rb.insert(tr)
    for tr in trs[:20]:
        demo.insert(tr)
    agent = make_drq_agent(42, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu")
    it = rb.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    dit = demo.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    del dry[:]
    batch = concat_batches(next(it), next(dit), axis=0)             # RLPD 50/50
    assert batch.batch_size == 8
    agent, info = agent.update_critics(batch)
    assert set(info) == {"critic", "critic_lr", "actor_lr", "temperature_lr"}
    assert set(info["critic"]) == {"critic_loss", "predicted_qs", "target_qs"}
    seq = [c for c in dry if c not in ("serl_replay_scatter", "serl_replay_set_valid", "serl_replay_commit")]     # pending inserts are flushed by sample()
    assert seq[0] == "serl_rng_schedule" and seq.count("serl_replay_sample_crop") == 2       # online + demo halves
    assert seq.count("serl_conv2d_nhwc_f32") == 2 * 12                                       # 12 convs per camera, ONE trunk pass
    assert seq.count("serl_adam_polyak") == 1 and seq[-1] == "serl_adam_polyak"
    assert agent.kernel_launches > 100
    del dry[:]
    agent, info = agent.update_high_utd(next(it).concat(next(dit)), utd_ratio=1)
    assert set(info["actor"]) == {"actor_loss", "temperature", "entropy"} and "temperature_loss" in info["temperature"]
    seq = list(dry)
    assert seq.count("serl_adam_polyak") == 2 and seq.count("serl_rng_schedule") == 3        # aug, critic update, actor/temp update
    assert seq.count("serl_conv2d_nhwc_f32") == 2 * 12                                       # features reused by actor/temperature
    assert seq.count("serl_actor_loss") == 1 and seq.count("serl_temperature_loss") == 1 and seq.count("serl_critic_loss") == 1
    assert agent.state.step == 3
    # wire format: Flax-layout tree incl. the frozen trunk
    tree = agent.state.params
    enc = tree["modules_actor"]["encoder"]
    assert enc["encoder_front"]["pretrained_encoder"]["conv_init"]["kernel"].shape == (7, 7, 3, 64)
    assert enc["encoder_wrist"]["SpatialLearnedEmbeddings_0"]["kernel"].shape == (4, 4, 512, 8)
    assert tree["modules_critic"]["network"]["Dense_0"]["kernel"].shape == (10, 256 * 2 + 64 + 4, 256)
    assert tree["modules_critic"]["Dense_0"]["kernel"].shape == (256, 1)
    assert tree["modules_temperature"]["lagrange"].shape == ()
    agent.state.replace(params=tree)


def test_state_sac_high_utd_and_sample_actions(dry):
    from serl_b200.utils.launcher import make_sac_agent
    rng = np.random.default_rng(0)
    agent = make_sac_agent(0, rng.standard_normal(10).astype(np.float32), np.zeros(4, np.float32), device="cpu")
    B = 32
    batch = dict(observations=rng.standard_normal((B, 10)).astype(np.float32), next_observations=rng.standard_normal((B, 10)).astype(np.float32),
                 actions=np.zeros((B, 4), np.float32), rewards=np.zeros(B, np.float32), masks=np.ones(B, np.float32), dones=np.zeros(B, bool))
    del dry[:]
    agent, info = agent.update_high_utd(batch, utd_ratio=4)
    assert dry.count("serl_adam_polyak") == 5 and dry.count("serl_critic_loss") == 4 and "serl_conv2d_nhwc_f32" not in dry
    assert agent.state.step == 5
    a = agent.sample_actions(rng.standard_normal(10).astype(np.float32), argmax=True)
    assert a.shape == (4,)
    a = agent.sample_actions(rng.standard_normal((3, 10)).astype(np.float32), seed=np.array([0, 7], np.uint32))
    assert a.shape == (3, 4)
    tree = agent.state.params
    assert tree["modules_critic"]["Dense_0"]["kernel"].shape == (10, 256, 1)
    os_ = agent.state.opt_states
    assert set(os_) == {"actor", "critic", "temperature"} and os_["actor"]["count"] == 0    # counts live on the (dry) device


def test_bf16_trunk_call_sequence(dry):
    from serl_b200.utils.launcher import make_drq_agent
    cams = ("front",)
    rb = _ring(cams, 64, 128)
    trs = random_transitions(np.random.default_rng(0), 40, cams, 128)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu",
                           precision="bf16")
    del dry[:]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    # 12 convs in 9 launches: the stem (fused with its max-pool), 5 stride-1 3x3 convs with GroupNorm (+ residual) + ReLU inside
    # (conv3x3_res), 3 stage heads = stride-2 3x3 conv + 1x1 projection + both GroupNorms in one kernel (conv3x3s2_res)
    assert dry.count("serl_stem_conv_pool_tc_h16") == 1 and dry.count("serl_pool_finish_gn_h16") == 1
    assert dry.count("serl_conv3x3_res_h16") == 5 and dry.count("serl_conv3x3s2_res_h16") == 3
    assert dry.count("serl_conv2d_tc_h16") == 0 and dry.count("serl_conv2d_nhwc_f32") == 0
    # no GroupNorm / residual pass of its own
    assert dry.count("serl_gn_finalize") == 0
    assert dry.count("serl_trunk_stem_prep_h16") == 1 and dry.count("serl_maxpool_affine_h16") == 0
    trunk = {"serl_trunk_stem_prep_h16", "serl_stem_conv_pool_tc_h16", "serl_pool_finish_gn_h16", "serl_conv3x3_res_h16", "serl_conv3x3s2_res_h16"}
    assert {n for n in dry if n.endswith("_h16")} == trunk
    assert dry.count("serl_gemm_tf32x3") > 0 and dry.count("serl_gemm_f32") == 0      # 16-bit builds: tensor-core heads


@pytest.mark.parametrize("hw", [64, 256])
@pytest.mark.parametrize("precision", ["fp32", "bf16", "fp16"])
def test_frozen_trunk_refuses_frames_other_than_128(dry, hw, precision):
    """The trunk divides a frame by 32 into the (4, 4, 512) features its consumers allocate: other frame sizes are refused where
    the trunk is built, for DrQ ("resnet-pretrained"), BC and the trunk itself."""
    from serl_b200.trunk import FrozenTrunk
    from serl_b200.utils.launcher import make_bc_agent, make_drq_agent
    cams = ("front",)
    tr = random_transitions(np.random.default_rng(0), 1, cams, hw)[0]
    for make in (make_drq_agent, make_bc_agent):
        with pytest.raises(NotImplementedError, match="128x128"):
            make(1, tr["observations"], tr["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu", precision=precision)
    with pytest.raises(NotImplementedError, match="128x128"):
        FrozenTrunk({"front": {}}, precision, hw)
    FrozenTrunk({}, precision, hw)                                  # state-only agents: no cameras, nothing to encode


def test_conv_tc_refuses_non_stem_descriptors():
    """serl_conv2d_tc_h16 is the unfused stem only: any other convolution is refused on the host, before a launch."""
    import ctypes as C
    from serl_b200 import _lib as L
    lib = L.load()
    d = L.ConvTcDesc()
    d.x = d.w = d.y = d.stats = d.error = 16                        # never dereferenced: the descriptor is refused first
    d.N, d.Hi, d.Wi, d.Ci, d.Ho, d.Wo, d.Co, d.kh, d.kw, d.stride, d.pad_lo, d.stem, d.fmt = 4, 32, 32, 64, 32, 32, 64, 3, 3, 1, 1, 0, L.FMT_FP16
    assert lib.serl_conv2d_tc_h16(C.byref(d), None) == -3                # SERL_ERR_UNSUPPORTED
    assert "only the stem" in lib.serl_last_error().decode()


def test_fused_heads_call_sequence(dry, monkeypatch):
    """Host logic of the fused critic step (heads_fused.py) on the dry device: launch counts per kernel family for two cameras."""
    monkeypatch.setenv("SERL_FUSED_HEADS", "force")
    from serl_b200.utils.launcher import make_drq_agent
    cams = ("front", "wrist")
    rb = _ring(cams, 64, 128)
    trs = random_transitions(np.random.default_rng(0), 40, cams, 128)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu",
                           precision="fp16")
    del dry[:]
    agent.update_critics(rb.sample(4, pack_obs_and_next_obs=True))
    # forward: 1 SLE + 1 k-split GEMM + 1 finish for the 3 passes x 2 cameras, 2 policy GEMMs, 2 critic GEMMs (online + target per layer);
    # backward: dh1, d enc, dW2, dW1, encoder dW, d SLE
    assert dry.count("serl_sle_fwd_multi") == 1 and dry.count("serl_enc_finish") == 1 and dry.count("serl_sle_fwd") == 0
    assert dry.count("serl_tgemm_tf32") == 1 + 2 + 2 + 6
    assert dry.count("serl_layernorm_tanh_bwd_multi") == 3 and dry.count("serl_small_grads") == 2
    assert dry.count("serl_layernorm_tanh_fwd") == 0 and dry.count("serl_colsum_f32") == 0
    assert dry.count("serl_gemm_tf32x3") == 1                                  # the (S, 64) proprio weight gradient: fan-in not TMA-addressable
    assert dry.count("serl_critic_loss") == 1 and dry.count("serl_adam_polyak") == 1


def test_pipelined_update_critics_call_sequence(dry):
    """Host logic of the cross-step pipeline: the first call of a handle sequence runs two front ends (its own + the next step's),
    every following sequential call runs one (the next step's) next to its heads; a call that breaks the sequence starts over."""
    from serl_b200.utils.launcher import make_drq_agent
    cams = ("front",)
    rb = _ring(cams, 64, 128)
    trs = random_transitions(np.random.default_rng(0), 40, cams, 128)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu",
                           precision="fp16")
    agent.pipeline_critic_steps = True
    agent._graph_key = lambda tag, batch: ("dry",)                  # the dry device cannot capture graphs: pipelined path, eager bodies
    agent.use_cuda_graphs = False
    it = rb.get_iterator(sample_args={"batch_size": 4, "pack_obs_and_next_obs": True})
    counts = []
    for _ in range(3):
        del dry[:]
        agent.update_critics(next(it))
        counts.append((dry.count("serl_replay_sample_crop"), dry.count("serl_stem_conv_pool_tc_h16"), dry.count("serl_critic_loss"), dry.count("serl_rng_schedule")))
    assert counts == [(2, 2, 1, 2), (1, 1, 1, 1), (1, 1, 1, 1)]
    assert agent.state.step == 3
    next(it)                                                        # skip a handle: the prefetched batch is not the next one
    del dry[:]
    agent.update_critics(next(it))
    assert dry.count("serl_replay_sample_crop") == 2 and dry.count("serl_critic_loss") == 1
    del dry[:]
    agent.update_high_utd(next(it), utd_ratio=1)                    # another entry point drops the prefetch
    agent.update_critics(next(it))
    assert dry.count("serl_replay_sample_crop") == 1 + 2


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_bc_agent_call_sequence(dry, precision):
    """Host logic of BCAgent.update / sample_actions (SURVEY.md §8 f4): one trunk pass per camera, the image heads are forward-only
    (stop_gradient), the proprio encoder and the tanh MLP (no LayerNorm) are differentiated, one Adam."""
    from serl_b200.utils.launcher import make_bc_agent
    cams = ("front", "wrist")
    trs = random_transitions(np.random.default_rng(0), 6, cams, 128)
    agent = make_bc_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu", precision=precision)
    batch = {"observations": {**{c: np.stack([t["observations"][c] for t in trs]) for c in cams}, "state": np.stack([t["observations"]["state"] for t in trs])},
             "actions": np.stack([t["actions"] for t in trs]).astype(np.float32)}
    rng0 = agent.state.rng
    del dry[:]
    agent, info = agent.update(batch)
    assert set(info) == {"actor_loss", "mse"} and agent.state.step == 1 and not np.array_equal(agent.state.rng, rng0)
    assert dry.count("serl_sle_fwd") == 2 and dry.count("serl_dropout_mask_fill") == 2 and dry.count("serl_bc_loss") == 1
    assert dry.count("serl_tanh_fwd") == 2 and dry.count("serl_tanh_bwd") == 2 and dry.count("serl_adam_polyak") == 1
    assert dry.count("serl_layernorm_tanh_fwd") == 3 and dry.count("serl_layernorm_tanh_bwd") == 1      # heads forward; only the proprio LN backward
    gemm = "serl_gemm_f32" if precision == "fp32" else "serl_gemm_tf32x3"
    assert dry.count(gemm) == (2 + 1 + 4) + (2 + 2 + 1 + 1 + 1 + 1 + 1)        # forward: 2 image heads, proprio, 4 policy; backward: head dW x2, head dX x2, dW2, dh1, dW1, d proprio, dW proprio
    tree = agent.state.params
    assert tree["modules_actor"]["network"]["Dense_0"]["kernel"].shape == (256 * 2 + 64, 256) and "LayerNorm_0" not in tree["modules_actor"]["network"]
    a = agent.sample_actions({k: v[0] for k, v in batch["observations"].items()}, argmax=True)
    assert a.shape == (4,)
    a = agent.sample_actions(batch["observations"], seed=np.array([0, 3], np.uint32))
    assert a.shape == (6, 4)
    agent.state.replace(params=tree)


def test_fused_actor_temperature_call_sequence(dry, monkeypatch):
    """Host logic of the fused actor / temperature step (heads_fused.py): encoder passes of both losses in one SLE / GEMM / finish
    launch each, one launch per policy layer for both policy passes, critic forward + dQ/da on the TF32 GEMMs."""
    monkeypatch.setenv("SERL_FUSED_HEADS", "force")
    from serl_b200.utils.launcher import make_drq_agent
    cams = ("front", "wrist")
    rb = _ring(cams, 64, 128)
    trs = random_transitions(np.random.default_rng(0), 40, cams, 128)
    for tr in trs:
        rb.insert(tr)
    agent = make_drq_agent(1, trs[0]["observations"], trs[0]["actions"], image_keys=cams, encoder_type="resnet-pretrained", device="cpu", precision="fp16")
    del dry[:]
    agent, info = agent.update_high_utd(rb.sample(4, pack_obs_and_next_obs=True), utd_ratio=1)
    assert set(info) >= {"critic", "actor", "temperature"}
    assert dry.count("serl_sle_fwd_multi") == 2 and dry.count("serl_enc_finish") == 2                  # critic step + actor / temperature step
    assert dry.count("serl_actor_loss") == 1 and dry.count("serl_temperature_loss") == 1 and dry.count("serl_critic_loss") == 1
    assert dry.count("serl_tgemm_tf32") == 11 + (1 + 2 + 2 + 2)                                        # + encoder GEMM, 2 policy layers, 2 critic layers, dh1, dQ/da
    assert dry.count("serl_layernorm_tanh_fwd") == 0 and dry.count("serl_sle_fwd") == 0
    assert dry.count("serl_adam_polyak") == 2 and agent.state.step == 2
