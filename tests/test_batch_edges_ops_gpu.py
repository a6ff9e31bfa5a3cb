"""GPU: the head kernels op by op at the batch sizes where their tiling, k-splits, chunking or row loops change, against
float64 restatements on the same fp32 inputs, and two launches of each bitwise equal.

At B ~ 2048 a lost or double-counted row moves a whole gradient leaf by about 1/B of its max, close to the agent-level
tests' 2e-4 bar; here one row is far above each op's bar.  Bars are the ones of tests/test_ops_gpu.py (fp32-class kernels,
2e-5), tests/test_heads_fused_ops_gpu.py (2e-5) and tests/test_tgemm_gpu.py (single-pass TF32, 2e-3).  Regimes:
  tgemm                weight-gradient layout (k = rows) at R in {1, 31, 33, 129, 200, 257, 1025, 2048}: 32-row k-blocks with
                       1- and 31-row tails; the PARTIAL epilogue + serl_enc_finish at the heads' k-split for 1, 129, 257 and
                       1024 rows; the LayerNorm-tanh epilogue with 1-row M tiles.
  gemm_f32, tf32x3     M or K in {1, 63, 64, 127, 128, 129, 390, 704, 705, 2048}, Z in {1, 10}: split-K on either side of
                       tiles < 448 / < 132 and K >= 128 (gemm_f32 at K = 390 leaves its last of six splits empty), and a
                       workspace that caps S.
  sle_bwd_multi        N in {1, 63, 64, 65, 1024, 2048}: 1 chunk below 64 rows, 16 from 64; fewer chunks in a short workspace.
  small_grads, colsum  rows in {1, 31, 33, 127, 129, 2561, 20480}: 4 x 32 rows in flight, then the 32-row tail; 8 row slices.
  SAC losses           B in {1, 1023, 1024, 1025, 2048, 4096}: one 1024-thread block, several rows per thread from 1025."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 2e-5          # fp32 kernels (tests/test_ops_gpu.py, tests/test_heads_fused_ops_gpu.py)
TGEMM_TOL = 2e-3    # single-pass TF32 (tests/test_tgemm_gpu.py)
ROWS = [1, 63, 64, 127, 128, 129, 390, 704, 705, 2048]


def cu(x, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(x)).cuda()
    return t if dt is None else t.to(dt)


def rel_err(a, b):
    b = np.asarray(b, np.float64)
    return float(np.max(np.abs(np.asarray(a, np.float64) - b)) / (np.max(np.abs(b)) + 1e-30))


def _twice(launch, *outs):
    """launch() twice, into outputs filled with the same sentinel; every output bitwise equal between the two; returns the outputs
    as float64 host arrays."""
    for o in outs:
        o.fill_(-7.0)
    launch()
    first = [o.clone() for o in outs]
    for o in outs:
        o.fill_(-7.0)
    launch()
    for a, b in zip(first, outs):
        assert torch.equal(a, b), "two launches differ"
    return [o.cpu().numpy().astype(np.float64) for o in outs]


def _ln_tanh(z, sc, lb, eps=1e-6):
    mean = z.mean(-1, keepdims=True)
    var = np.maximum((z * z).mean(-1, keepdims=True) - mean * mean, 0.0)
    return np.tanh((z - mean) / np.sqrt(var + eps) * sc + lb)


# ---- tgemm --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 31, 33, 129, 200, 257, 1025, 2048])
def test_tgemm_weight_gradient_rows(R):
    """dW (fan_in, 256) = X^T dZ with k = R batch rows, at fan-in 4096 (encoder), 580 (critic layer 0, 10 members), 256."""
    from serl_b200 import ops
    rng = np.random.default_rng(R)
    ws = ops.Workspace(64 << 20, "cuda")
    for FI, Z in ((4096, 1), (580, 10), (256, 10)):
        x = rng.standard_normal((R, FI)).astype(np.float32)
        dz = rng.standard_normal((Z, R, 256)).astype(np.float32)
        xd, dzd = cu(x), cu(dz)
        dw = torch.zeros(Z, FI, 256, device="cuda")
        p = ops.tgemm_problem(xd.data_ptr(), dzd.data_ptr(), sAm=1, sAk=FI, sBk=256, sBn=1, Z=Z, sBz=R * 256, C_=dw.data_ptr(),
                              sCz=FI * 256, ldc=256)
        got, = _twice(lambda: ops.tgemm(ws, [p], FI, 256, R), dw)
        e = rel_err(got, np.einsum("rk,zrn->zkn", x.astype(np.float64), dz.astype(np.float64)))
        print(f"tgemm wgrad R={R} fan_in={FI} Z={Z}: {e:.2e}")
        assert e < TGEMM_TOL, (FI, Z, e)


@pytest.mark.parametrize("M", [1, 129, 257, 1024])
def test_tgemm_partial_and_enc_finish_at_heads_split(M):
    """The encoder Dense 4096 -> 256 as the fused heads run it: two problems (cameras) in one PARTIAL launch at the heads'
    k-split for two cameras x three passes, then serl_enc_finish sums the S partials and applies bias + LayerNorm + tanh."""
    from serl_b200 import _lib as L
    from serl_b200 import ops
    rng = np.random.default_rng(M + 1)
    S = ops.tgemm_splits(4096, max(1, min(132 // (6 * ((M + 127) // 128)), 32)))
    assert S == {1: 22, 129: 11, 257: 7, 1024: 2}[M]
    ws = ops.Workspace(2 * S * M * 256 * 4, "cuda")
    x = np.abs(rng.standard_normal((2, M, 4096))).astype(np.float32)
    w = (rng.standard_normal((2, 4096, 256)) / 64).astype(np.float32)
    b, lb = [(0.2 * rng.standard_normal((2, 256))).astype(np.float32) for _ in range(2)]
    sc = (1 + 0.2 * rng.standard_normal((2, 256))).astype(np.float32)
    t = {k: cu(v) for k, v in dict(x=x, w=w, b=b, sc=sc, lb=lb).items()}
    out = torch.zeros(M, 580, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    probs = [ops.tgemm_problem(t["x"].data_ptr() + 4 * i * M * 4096, t["w"].data_ptr() + 4 * i * 4096 * 256, sAm=4096, sAk=1, sBk=256, sBn=1)
             for i in range(2)]
    fin = [dict(partials=ws.buf.data_ptr() + 4 * i * S * M * 256, S=S, bias=t["b"].data_ptr() + 1024 * i, ln_scale=t["sc"].data_ptr() + 1024 * i,
                ln_bias=t["lb"].data_ptr() + 1024 * i, out=ops.at(out, 256 * i), ld_out=580, D=256) for i in range(2)]

    def launch():
        ops.tgemm(ws, probs, M, 256, 4096, epilogue=L.TGEMM_PARTIAL, splits=S, error=err)
        ops.enc_finish(fin, M)
    got, = _twice(launch, out)
    assert int(err.item()) == 0
    for i in range(2):
        ref = _ln_tanh(x[i].astype(np.float64) @ w[i].astype(np.float64) + b[i], sc[i].astype(np.float64), lb[i].astype(np.float64))
        e = rel_err(got[:, 256 * i:256 * (i + 1)], ref)
        print(f"tgemm PARTIAL + enc_finish M={M} S={S} camera {i}: {e:.2e}")
        assert e < TGEMM_TOL, (i, e)


@pytest.mark.parametrize("M", [1, 129, 257])
def test_tgemm_ln_tanh_epilogue_rows(M):
    from serl_b200 import _lib as L
    from serl_b200 import ops
    rng = np.random.default_rng(M + 2)
    K = 580
    x = rng.standard_normal((M, K)).astype(np.float32)
    w = (rng.standard_normal((K, 256)) / np.sqrt(K)).astype(np.float32)
    b, lb = [(0.1 * rng.standard_normal(256)).astype(np.float32) for _ in range(2)]
    sc = (1 + 0.1 * rng.standard_normal(256)).astype(np.float32)
    t = {k: cu(v) for k, v in dict(x=x, w=w, b=b, sc=sc, lb=lb).items()}
    h = torch.zeros(M, 256, device="cuda")
    p = ops.tgemm_problem(t["x"].data_ptr(), t["w"].data_ptr(), sAm=K, sAk=1, sBk=256, sBn=1, C_=h.data_ptr(), ldc=256, bias=t["b"].data_ptr(),
                          ln_scale=t["sc"].data_ptr(), ln_bias=t["lb"].data_ptr())
    got, = _twice(lambda: ops.tgemm(None, [p], M, 256, K, epilogue=L.TGEMM_LN_TANH), h)
    e = rel_err(got, _ln_tanh(x.astype(np.float64) @ w.astype(np.float64) + b, sc.astype(np.float64), lb.astype(np.float64)))
    print(f"tgemm LN-tanh M={M}: {e:.2e}")
    assert e < TGEMM_TOL


# ---- per-op GEMMs -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", ["f32", "tf32x3"])
@pytest.mark.parametrize("R", ROWS)
def test_dense_ops_rows(R, impl):
    """Forward (M = R rows), weight gradient (K = R rows) and input gradient (M = R, reduced over members when Z = 10) of a
    critic layer (580 -> 256) and the single-member policy head (256 -> 256)."""
    from serl_b200 import ops
    rng = np.random.default_rng(R + 3)
    ws = ops.Workspace(64 << 20, "cuda", impl)
    for K, N, Z in ((580, 256, 10), (256, 256, 1)):
        x = rng.standard_normal((Z, R, K)).astype(np.float32)
        w = (rng.standard_normal((Z, K, N)) / np.sqrt(K)).astype(np.float32)
        b = rng.standard_normal((Z, N)).astype(np.float32)
        dz = rng.standard_normal((Z, R, N)).astype(np.float32)
        xd, wd, bd, dzd = cu(x), cu(w), cu(b), cu(dz)
        x64, w64, dz64 = x.astype(np.float64), w.astype(np.float64), dz.astype(np.float64)
        out, dw = torch.empty(Z, R, N, device="cuda"), torch.empty(Z, K, N, device="cuda")
        dx = torch.empty(R, K, device="cuda") if Z > 1 else torch.empty(1, R, K, device="cuda")
        got_out, = _twice(lambda: ops.dense_fwd(ws, xd.data_ptr(), K, wd.data_ptr(), bd.data_ptr(), out.data_ptr(), N, R, K, N, Z=Z,
                                                x_z=R * K, out_z=R * N), out)
        got_dw, = _twice(lambda: ops.dense_bwd_weight(ws, xd.data_ptr(), K, dzd.data_ptr(), N, dw.data_ptr(), R, K, N, Z=Z, x_z=R * K,
                                                      dz_z=R * N), dw)
        got_dx, = _twice(lambda: ops.dense_bwd_input(ws, dzd.data_ptr(), N, wd.data_ptr(), dx.data_ptr(), K, R, K, N, Z=Z, dz_z=R * N,
                                                     reduce_z=Z > 1), dx)
        errs = {"fwd": rel_err(got_out, np.einsum("zmk,zkn->zmn", x64, w64) + b[:, None, :]),
                "wgrad": rel_err(got_dw, np.einsum("zmk,zmn->zkn", x64, dz64)),
                "dgrad": rel_err(got_dx.reshape(R, K), np.einsum("zmn,zkn->mk", dz64, w64))}
        print(f"{impl} R={R} K={K} Z={Z}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
        assert all(v < TOL for v in errs.values()), (K, Z, errs)


@pytest.mark.parametrize("impl", ["f32", "tf32x3"])
def test_dense_weight_gradient_with_capped_workspace(impl):
    """2048 rows into a 256 x 256 weight gradient wants 32 k-splits; a workspace of three partials caps S at 3."""
    from serl_b200 import ops
    rng = np.random.default_rng(17)
    R, K, N = 2048, 256, 256
    x = rng.standard_normal((R, K)).astype(np.float32)
    dz = rng.standard_normal((R, N)).astype(np.float32)
    xd, dzd = cu(x), cu(dz)
    ref = x.astype(np.float64).T @ dz.astype(np.float64)
    for parts in (3, 1):
        ws = ops.Workspace(parts * K * N * 4 + 4, "cuda", impl)
        dw = torch.empty(K, N, device="cuda")
        got, = _twice(lambda: ops.dense_bwd_weight(ws, xd.data_ptr(), K, dzd.data_ptr(), N, dw.data_ptr(), R, K, N), dw)
        e = rel_err(got, ref)
        print(f"{impl} capped workspace ({parts} partials): {e:.2e}")
        assert e < TOL, (parts, e)


# ---- SLE kernel gradient ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 63, 64, 65, 1024, 2048])
def test_sle_bwd_multi_rows(N):
    from serl_b200 import ops
    rng = np.random.default_rng(N + 4)
    per_chunk = 2 * 16 * 512 * 8 * 4
    feats = [np.abs(rng.standard_normal((N, 4, 4, 512))).astype(np.float32) for _ in range(2)]
    douts = [rng.standard_normal((N, 4096)).astype(np.float32) for _ in range(2)]
    fd, dd = [cu(f) for f in feats], [cu(d) for d in douts]
    outs = [torch.zeros(4, 4, 512, 8, device="cuda") for _ in range(2)]
    refs = [np.einsum("bhwc,bcf->hwcf", f.astype(np.float64), d.astype(np.float64).reshape(N, 512, 8)) for f, d in zip(feats, douts)]
    probs = [(f.data_ptr(), d.data_ptr(), 4096, o.data_ptr()) for f, d, o in zip(fd, dd, outs)]
    for chunks in (16, 4):                                             # a workspace of 16 chunks, then one of 4
        ws = ops.Workspace(chunks * per_chunk, "cuda")
        got = _twice(lambda: ops.sle_bwd_multi(ws, probs, N, 16, 512), *outs)
        for i, (g, r) in enumerate(zip(got, refs)):
            e = rel_err(g, r)
            print(f"sle_bwd_multi N={N} workspace {chunks} chunks camera {i}: {e:.2e}")
            assert e < TOL, (chunks, i, e)


# ---- column reductions --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 31, 33, 127, 129, 2561, 20480])
def test_small_grads_and_colsum_rows(rows):
    from serl_b200 import _lib as L
    from serl_b200 import ops
    rng = np.random.default_rng(rows + 5)
    G, D = 2, 256
    x = rng.standard_normal((G * rows, D)).astype(np.float32)
    y = rng.standard_normal((G * rows, D)).astype(np.float32)
    dq = rng.standard_normal(G * rows).astype(np.float32)
    T = {k: cu(v) for k, v in dict(x=x, y=y, dq=dq).items()}
    cs, la, lb = (torch.zeros(G, D, device="cuda") for _ in range(3))
    hw, hb, col = torch.zeros(D, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(G, D, device="cuda")
    jobs = [(L.SMALL_GRAD_COLSUM, T["x"].data_ptr(), D, None, 0, cs.data_ptr(), None, G, rows, D),
            (L.SMALL_GRAD_LN, T["x"].data_ptr(), D, T["y"].data_ptr(), D, la.data_ptr(), lb.data_ptr(), G, rows, D),
            (L.SMALL_GRAD_HEAD, T["x"].data_ptr(), D, T["dq"].data_ptr(), 1, hw.data_ptr(), hb.data_ptr(), 1, G * rows, D)]
    g_cs, g_la, g_lb, g_hw, g_hb = _twice(lambda: ops.small_grads(jobs), cs, la, lb, hw, hb)
    g_col, = _twice(lambda: ops.colsum(T["x"].data_ptr(), col.data_ptr(), G, rows, D, D), col)
    x64, y64, dq64 = x.astype(np.float64).reshape(G, rows, D), y.astype(np.float64).reshape(G, rows, D), dq.astype(np.float64)
    errs = {"colsum job": rel_err(g_cs, x64.sum(1)), "ln job a": rel_err(g_la, (x64 * y64).sum(1)), "ln job b": rel_err(g_lb, x64.sum(1)),
            "head job w": rel_err(g_hw, (x64.reshape(-1, D) * dq64[:, None]).sum(0)), "head job b": rel_err(g_hb, [dq64.sum()]),
            "colsum": rel_err(g_col, x64.sum(1))}
    print(f"reductions rows={rows}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v < TOL for v in errs.values()), errs


# ---- SAC losses ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 1023, 1024, 1025, 2048, 4096])
def test_sac_losses_rows(B):
    """critic_loss (per-row target and dQ, loss / mean Q / mean target), actor_loss (per-row dmu / dlog_std, loss / alpha /
    entropy) and temperature_loss, each in one 1024-thread block, against float64."""
    from serl_b200 import ops
    rng = np.random.default_rng(B + 6)
    E, A, gamma = 10, 4, 0.96
    lam64 = float(np.float32(-4.6))
    alpha = np.log1p(np.exp(lam64))
    lam = cu(np.array([lam64], np.float32))
    # critic loss, TD target from the min over a 2-member subsample
    q, qn = rng.standard_normal((E, B)).astype(np.float32), rng.standard_normal((E, B)).astype(np.float32)
    r, m = rng.random(B).astype(np.float32), (rng.random(B) > 0.1).astype(np.float32)
    logp = rng.standard_normal(B).astype(np.float32)
    sub = np.array([3, 7], np.int32)
    tq, dq, info = torch.empty(B, device="cuda"), torch.empty(E, B, device="cuda"), torch.zeros(4, device="cuda")
    qd, qnd, subd, rd, md, lpd = cu(q), cu(qn), cu(sub), cu(r), cu(m), cu(logp)
    g_tq, g_dq, g_info = _twice(lambda: ops.critic_loss(qd, qnd, subd, 2, rd, md, lpd, lam.data_ptr(), False, gamma, 1.0, tq, dq,
                                                        info.data_ptr(), E, B), tq, dq, info)
    q64 = q.astype(np.float64)
    y = r + gamma * m.astype(np.float64) * np.minimum(qn[3], qn[7]).astype(np.float64)
    errs = {"target_q": rel_err(g_tq, y), "dq": rel_err(g_dq, 2 * (q64 - y[None]) / (E * B)),
            "critic_loss": rel_err(g_info[:1], [((q64 - y[None]) ** 2).mean()]), "mean q": abs(g_info[1] - q64.mean()) / (abs(q64.mean()) + 0.1),
            "mean target": rel_err(g_info[2:3], [y.mean()])}
    # actor loss (exp std parameterisation; a few entries on each std clip)
    mu_da = rng.standard_normal((B, A)).astype(np.float32) / B
    act = np.tanh(rng.standard_normal((B, A))).astype(np.float32)
    ls = (rng.standard_normal((B, A)) * 1.5).astype(np.float32)
    ls.reshape(-1)[::97] = 3.0
    ls.reshape(-1)[1::97] = -14.0
    std = np.clip(np.exp(ls.astype(np.float64)), 1e-5, 5.0).astype(np.float32)
    eps = rng.standard_normal((B, A)).astype(np.float32)
    dmu, dls, ainfo = torch.empty(B, A, device="cuda"), torch.empty(B, A, device="cuda"), torch.zeros(4, device="cuda")
    dad, actd, stdd, lsd, epsd = cu(mu_da), cu(act), cu(std), cu(ls), cu(eps)
    g_dmu, g_dls, g_ainfo = _twice(lambda: ops.actor_loss(qd, lpd, lam.data_ptr(), dad.data_ptr(), A, actd.data_ptr(), A, stdd, lsd, epsd,
                                                          1e-5, 5.0, 1.0, dmu, dls, ainfo.data_ptr(), E, B, A), dmu, dls, ainfo)
    a64, std64, eps64 = act.astype(np.float64), std.astype(np.float64), eps.astype(np.float64)
    du = mu_da.astype(np.float64) * (1 - a64 ** 2) + (alpha / B) * 2 * a64
    raw = np.exp(ls.astype(np.float32)).astype(np.float64)
    inside = (raw >= 1e-5) & (raw <= 5.0)
    obj = q64.mean(0) - alpha * logp.astype(np.float64)
    errs.update({"dmu": rel_err(g_dmu, du), "dlog_std": rel_err(g_dls, np.where(inside, du * std64 * eps64 - alpha / B, 0.0)),
                 "actor_loss": abs(g_ainfo[0] + obj.mean()) / (abs(obj.mean()) + 0.1), "alpha": rel_err(g_ainfo[1:2], [alpha]),
                 "entropy": abs(g_ainfo[2] + logp.astype(np.float64).mean()) / (abs(logp.astype(np.float64).mean()) + 0.1)})
    # temperature loss
    dl, ti = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    g_dl, g_ti = _twice(lambda: ops.temperature_loss(lpd, lam.data_ptr(), -2.0, 1.0, dl.data_ptr(), ti.data_ptr(), B), dl, ti)
    ent = -logp.astype(np.float64).mean()
    errs.update({"temperature_loss": rel_err(g_ti, [alpha * (ent + 2.0)]),
                 "dlagrange": rel_err(g_dl, [(ent + 2.0) / (1 + np.exp(-lam64))])})
    print(f"SAC losses B={B}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    assert all(v < TOL for v in errs.values()), errs
