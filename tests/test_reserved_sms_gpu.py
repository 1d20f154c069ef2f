"""The training kernels and both engines with SMs reserved for the overlapped gradient all-reduce.

A data-parallel step runs its last backward between DataParallel.begin_overlap() and wait(): db200_set_reserved_sms(k)
with k = MAX_CTAS (4 at >= 16 k tokens per GPU, 16 below), and with recompute_grad the recomputed block forward runs
there too.  sm_count() then returns max(SMs - k, 16), and every host launch rule that reads it changes: the persistent
GEMM / convolution grids, the split-K count of the weight gradients, the conv_tc pixel splits, the LayerNorm backward
grid (the chain lengths of dg / db / dxsum), the colsum, embed_bwd and cast grids.

The cases are those of test_dalle_kernels_gpu.py and test_vae_kernels_gpu.py, replayed through their helpers inside
float64_bounds.reserved_sms(k): the bounds follow the reserved count through float64_bounds.sm_count(), and every case
line starts with `[reserved-sms k=<k> sm=<n>]`.  k = 16 and 4 are the two defaults of the CTA cap; k = 5 leaves 127
SMs on a 132-SM H100 (prime: no tile count divides evenly); k = 64 is the largest reservation the library accepts.

Each test also shows that the reservation changed what runs (a split count, or for products that never split, the
tiles the busiest CTA walks), so it cannot pass on the unreserved grid; and an autouse fixture asks the library after
every test that nothing is reserved any more.

On an H100 80GB HBM3 (132 SMs, 400 W power limit) the module takes 33 s of wall time including start-up, against
19 s for test_dalle_kernels_gpu.py.
"""
import ctypes

import pytest
import torch

import float64_bounds
import test_dalle_kernels_gpu as DK
import test_engine_gpu as EG
import test_vae_kernels_gpu as VK
from float64_bounds import reserved_sms, sm_count

pytestmark = pytest.mark.gpu

DALLE_CONFIGS = list(DK.CONFIGS)
VAE_CONFIGS = ["vae_example_b200", "vae_coco_b200"]


@pytest.fixture(scope="module")
def ops():
    from dalle_mtf_b200 import lib as L, ops as _ops
    L.require_device()
    return _ops


def device_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def line(k, sm, msg):
    print(f"[reserved-sms k={k} sm={sm}] {msg}")


def _cdiv(a, b):
    return -(-a // b)


def lib_splits(M, N, K, split_k=0):
    """The K splits the library runs for an ATOMIC product now: its workspace is one M x N fp32 slice per split."""
    from dalle_mtf_b200 import lib as L
    e = L.GemmEpilogue()
    e.mode, e.split_k = L.EPI_ATOMIC, split_k
    return max(1, L.load().db200_gemm_workspace_bytes(M, N, K, ctypes.byref(e)) // (M * N * 4))


def probe():
    """The SM count the library uses, read back through the split-K rule: one 128 x 128 tile over 4m k-blocks asks
    for min(SMs, m) slices.  With m = n = sm_count() the workspace is exactly n slices (the library sees no fewer
    SMs than n); with m = n + 1, n slices of 5 k-blocks cover them in ceil(4 (n + 1) / 5) splits, n + 1 SMs would
    give n + 1 splits of 4 (it sees no more)."""
    from dalle_mtf_b200 import lib as L
    n = sm_count()
    e = L.GemmEpilogue()
    e.mode, e.split_k = L.EPI_ATOMIC, 0
    got = L.load().db200_gemm_workspace_bytes(128, 128, 256 * n, ctypes.byref(e))
    assert got == n * 128 * 128 * 4, (float64_bounds.reservation(), n, got // (128 * 128 * 4))
    K = 256 * (n + 1)
    assert lib_splits(128, 128, K) == DK.gemm_splits(128, 128, K, L.EPI_ATOMIC, 0, n), (float64_bounds.reservation(), n)
    return n


@pytest.fixture(autouse=True)
def _nothing_stays_reserved(ops):
    """A failing case must not leave the following tests (and modules) running on a smaller grid."""
    yield
    assert float64_bounds.reservation() == 0
    assert probe() == device_sms()


# ------------------------------------------------------------------------------------------------------- the knob
@pytest.mark.parametrize("k", [0, 4, 5, 16, 64])
def test_the_reservation_reaches_the_library(ops, k):
    with reserved_sms(k) as sm:
        assert probe() == sm == max(device_sms() - k, 16)
        line(k, sm, f"probe: 128x128x{256 * sm} ATOMIC runs {sm} K splits")


def test_out_of_range_reservations_are_refused_and_change_nothing(ops):
    from dalle_mtf_b200 import lib as L
    for bad in (-1, 65):
        with pytest.raises(L.DB200Error):
            with reserved_sms(bad):
                pass
        assert float64_bounds.reservation() == 0 and probe() == device_sms()
    with reserved_sms(16) as sm:
        for bad in (-1, 65):
            with pytest.raises(L.DB200Error):
                with reserved_sms(bad):
                    pass
            assert float64_bounds.reservation() == 16 and probe() == sm
    line(16, sm, "k = -1 and k = 65 refused; the reservation in force stays")


def _replay_shape(desc, T_rec, T):
    M, N, K = desc[1:4]
    return (T if M == T_rec else M), N, (T if K == T_rec else K)


@pytest.mark.parametrize("config", DALLE_CONFIGS)
def test_library_split_counts_match_the_mirror(ops, config):
    """gemm.cu gemm_splits and its mirror DK.gemm_splits agree on every ATOMIC product of the engine at every k."""
    from dalle_mtf_b200 import lib as L
    calls, _, _, _, S = DK.engine_calls(ops, config)
    atomic = [c for c in calls if c[0] == "gemm" and c[6] == L.EPI_ATOMIC]
    assert atomic
    for k in (0, 4, 5, 16, 64):
        with reserved_sms(k) as sm:
            for desc in atomic:
                M, N, K = _replay_shape(desc, S, DK.CONFIGS[config])
                want = DK.gemm_splits(M, N, K, L.EPI_ATOMIC, desc[12], sm)
                assert lib_splits(M, N, K, desc[12]) == want, (config, k, M, N, K)
            line(k, sm, f"{config}: library split counts of {len(atomic)} ATOMIC products match the mirror")


# ------------------------------------------------------------------------------------------------------- DALL-E
def _gemm_products(ops, config, k, modes):
    """Replays the configuration's recorded GEMM products of `modes` at its tokens per GPU with k SMs reserved
    (plus the residual-dropout STORE when STORE is among them).  Returns per product (name, splits at k = 0, splits
    now, tiles the busiest CTA walks at k = 0, now); checks the library's split count against the replay's."""
    from dalle_mtf_b200 import lib as L
    calls, _, _, _, S = DK.engine_calls(ops, config)
    T, full = DK.CONFIGS[config], device_sms()
    gemms = [c for c in calls if c[0] == "gemm"]
    rows = []
    with reserved_sms(k) as sm:
        for i, desc in enumerate(gemms):
            mode = desc[6]
            if mode not in modes:
                continue
            M, N, K = _replay_shape(desc, S, T)
            mn = _cdiv(M, 128) * _cdiv(N, 128)
            s0 = DK.gemm_splits(M, N, K, mode, desc[12], full)
            _, tiles, _ = DK.run_gemm_case(ops, desc, S, T, seed=i, tag=f"{config} ")
            sk = tiles // mn
            if mode == L.EPI_ATOMIC:
                assert lib_splits(M, N, K, desc[12]) == sk, (config, k, M, N, K, sk)
            w0, wk = _cdiv(mn * s0, min(mn * s0, full)), _cdiv(tiles, min(tiles, sm))
            name = f"{DK._mode_name(mode)} {M}x{N}x{K}"
            rows.append((name, s0, sk, w0, wk))
            line(k, sm, f"{config} {name}: splits {s0} -> {sk}, tiles per CTA {w0} -> {wk}")
        if L.EPI_STORE in modes:
            wo = [c for c in gemms if c[6] == L.EPI_STORE and c[10] and c[3] == c[2] == DK._config(config)["n_embd"]]
            assert len(wo) == 1
            drop = L.make_dropout(0.1, 7, 3, L.dropout_site_attn_out(0), 0)
            DK.run_gemm_case(ops, wo[0], S, T, seed=99, dropout=drop, tag=f"{config} ")
    return rows


def _assert_paths_changed(config, k, rows):
    """A configuration with split-K products must run one of them with another split count than at k = 0; one whose
    products never split (12B: every product has more tiles than SMs) must walk more tiles per CTA somewhere."""
    if any(s0 > 1 or sk > 1 for _, s0, sk, _, _ in rows):
        assert any(s0 != sk for _, s0, sk, _, _ in rows), (config, k, rows)
    else:
        assert any(w0 != wk for _, _, _, w0, wk in rows), (config, k, rows)


GEMM_CASES = [(16, c) for c in DALLE_CONFIGS] + [(4, "dalle_example_b200"), (4, "dalle_12b_b200")]


@pytest.mark.parametrize("k,config", GEMM_CASES)
def test_gemm_products_under_reservation(ops, k, config):
    from dalle_mtf_b200 import lib as L
    rows = _gemm_products(ops, config, k, {L.EPI_STORE, L.EPI_ATOMIC, L.EPI_RELU_BWD})
    assert len(rows) == 15
    if k != 4:                       # k = 4 leaves the split counts of these shapes on a 132-SM H100 unchanged
        _assert_paths_changed(config, k, rows)


@pytest.mark.parametrize("k", [5, 64])
@pytest.mark.parametrize("config", ["dalle_example_b200", "dalle_coco_b200"])
def test_gradient_products_at_odd_reservations(ops, config, k):
    """The ATOMIC (split-K wgrad), RELU_BWD and CE_GRAD products, where split counts and ragged last splits move."""
    from dalle_mtf_b200 import lib as L
    rows = _gemm_products(ops, config, k, {L.EPI_ATOMIC, L.EPI_RELU_BWD})
    _assert_paths_changed(config, k, rows)
    with reserved_sms(k):
        DK.real_vocabulary_cross_entropy(ops, config, DK.CONFIGS[config])


@pytest.mark.parametrize("config", DALLE_CONFIGS)
def test_cross_entropy_under_reservation(ops, config):
    """CE_STATS -> ce_finish -> CE_GRAD with the fused bias colsum, at the real vocabulary, with 16 SMs reserved."""
    with reserved_sms(16):
        DK.real_vocabulary_cross_entropy(ops, config, DK.CONFIGS[config])


LN_CASES = [(16, c) for c in DALLE_CONFIGS] + [(4, "dalle_example_b200"), (4, "dalle_12b_b200")]


@pytest.mark.parametrize("k,config", LN_CASES)
def test_layernorm_under_reservation(ops, k, config):
    """LayerNorm forward + backward at the engine's width and tokens per GPU: the backward grid, and with it the rows
    each thread chains into dg / db / dxsum, follows the reserved SM count (the d = 4096 forward grid too)."""
    from dalle_mtf_b200 import lib as L
    d, rows = DK._config(config)["n_embd"], DK.CONFIGS[config]
    kind = "wide" if d == 4096 else "warp"
    with reserved_sms(k) as sm:
        grid = min(rows if d == 4096 else _cdiv(rows, 4), 4 * sm)
        grid0 = min(rows if d == 4096 else _cdiv(rows, 4), 4 * device_sms())
        line(k, sm, f"{config} LN backward grid {grid0} -> {grid}")
        assert grid != grid0 or grid == (rows if d == 4096 else _cdiv(rows, 4))
        DK.run_layernorm(ops, f"{config} LN {kind} rows={rows} d={d} +dres", rows, d, seed=d)
        DK.run_layernorm(ops, f"{config} LN {kind} rows={rows} d={d} no dres", rows, d, dres=False, seed=d + 1)
        if k == 16:
            drop = L.make_dropout(0.1, 9, 4, L.dropout_site_mlp_out(0), 1280)
            DK.run_layernorm(ops, f"{config} LN dropout rows={rows} d={d}", rows, d, dropout=drop, seed=d + 2)


@pytest.mark.parametrize("config", DALLE_CONFIGS)
def test_embedding_backward_under_reservation(ops, config):
    cfg = DK._config(config)
    calls, extra, V, _, S = DK.engine_calls(ops, config)
    d, T = cfg["n_embd"], DK.CONFIGS[config]
    g = DK._gen(V + T)
    ids = DK.synthetic_tokens(cfg, T // S, g)
    scale = extra["dx_std"] * S / T
    with reserved_sms(16):
        DK.run_embedding(ops, f"{config} embedding T={T} grad std {scale:.2g}", ids, V, d, scale, g)


# ------------------------------------------------------------------------------------------------------- VAE
@pytest.mark.parametrize("k", [4, 16])
@pytest.mark.parametrize("config", VAE_CONFIGS)
def test_vae_convolutions_under_reservation(ops, config, k):
    """Every convolution of the training step (bf16 on wgmma, fp32 on the three-way split or direct kernels) at a
    batch sized from the reserved SM count; the conv2d_wgrad_tc pixel split moves for at least one layer (on
    vae_coco's 512-channel layers to a single split)."""
    full = device_sms()
    with reserved_sms(k) as sm:
        batches = VK.production_convolutions(ops, config, several_splits=False)
    changed = 0
    for (kind, cin, cout, res, kk, stride, transposed, _), n in batches:
        c = ops.conv_desc(n, res, res, cin, cout, kk, kk, stride, transposed=transposed, act_f32=False)
        if not ops.conv_wgrad_tc_supported(c):
            continue
        s0 = VK.wgrad_split(n, res, cin, cout, kk, stride, transposed, full)[2]
        sk = VK.wgrad_split(n, res, cin, cout, kk, stride, transposed, sm)[2]
        changed += s0 != sk
        line(k, sm, f"{config} {kind} {cin}->{cout} @{res} N={n}: wgrad pixel splits {s0} -> {sk}")
    assert changed, (config, k)


@pytest.mark.parametrize("N,H,Cin,Cout,k,stride,transposed", VK.EDGE_GEOMETRIES)
def test_edge_convolutions_with_64_sms_reserved(ops, N, H, Cin, Cout, k, stride, transposed):
    with reserved_sms(64):
        VK.test_tensor_core_convolutions_at_edge_geometries(ops, N, H, Cin, Cout, k, stride, transposed)


# ------------------------------------------------------------------------------------------------------- engines
DROPOUT = ((0.1, 0.2, 0.15), 11, 6, 1)          # (embed, attention, residual) rates, seed, step, row0
# a case may end in (attention_types, radius): the last one has a local layer (no attention dropout there)
ENGINE_CASES = [(c[:8], c[8], None) for c in EG.DALLE_CASES] + [(EG.DALLE_CASES[2][:8], True, DROPOUT),
                                                                 (EG.DALLE_CASES[2][:8] + (("global", "local"), 100),
                                                                  True, DROPOUT)]


@pytest.mark.parametrize("k", [4, 16])
@pytest.mark.parametrize("case,recompute,dropout", ENGINE_CASES)
def test_dalle_step_with_the_backward_under_reservation(ops, case, recompute, dropout, k):
    """As train_op runs it: forward with every SM, backward (and with recompute_grad the recomputed block forward)
    with k reserved, the optimiser step after the reservation ends; the criteria of
    test_dalle_forward_backward_optimizer_match_oracle."""
    EG.dalle_step_matches_oracle(case[:8], recompute, lambda: reserved_sms(k), dropout=dropout,
                                 local=case[8:] or None)
    line(k, max(device_sms() - k, 16), f"DalleEngine {case} recompute={recompute} dropout={dropout is not None}: "
         "forward / backward / optimizer step match the oracle")


def test_dalle_steps_are_bitwise_reproducible_under_reservation(ops):
    EG.training_steps_are_bitwise_reproducible(lambda: reserved_sms(16))
    line(16, max(device_sms() - 16, 16), "three DalleEngine steps bitwise identical across two runs")


def test_vae_bf16_step_with_the_backward_under_reservation(ops):
    EG.vae_bf16_step_matches_oracle(lambda: reserved_sms(4))
    line(4, max(device_sms() - 4, 16), "VaeEngine bf16 step: loss and gradients match the oracle")
