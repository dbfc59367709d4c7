"""Weight-only int8 on the GPU: b200mix_quantize_w8 against the CPU oracle bit for bit, b200mix_linear_w8 on both paths
against the fp32 oracle A @ (q * scale)^T + epilogue, and the tiny Qwen2-VL / Llama with quant_type="weight_only_int8"
against the fp32 oracles on the dequantized weights. Stated tolerance: the GEMM tolerance of the bf16 linear tests;
cosine >= 0.999 and max |err| <= 4 % of the logit range for the models."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import llama as OL
from oracle import qwen2vl as O
from oracle.quant import dequantize, dequantize_decoder_params, weight_quantize

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
GEMM_RTOL, GEMM_ATOL = 1.0e-2, 2e-2
ERR_INVALID, ERR_UNSUPPORTED = -1, -4
SMALL_MAX = 64  # W8_SMALL_MAX in linear_w8.cu


@pytest.fixture(scope="module")
def ops():
    from paddlemix_b200 import ops as _ops
    from paddlemix_b200._lib import lib
    _ops.init(0)
    lib.b200mix_debug_w8_small_max.argtypes, lib.b200mix_debug_w8_small_max.restype = [ctypes.c_int], None
    lib.b200mix_debug_skinny_splits.argtypes, lib.b200mix_debug_skinny_splits.restype = [ctypes.c_int], None
    return _ops


def unlayout(q: torch.Tensor, N: int, K: int) -> torch.Tensor:
    """The device layout of b200mix_quantize_w8 ([N/16][K/32][lane 4g+t][byte 8s+2r+e], r = 2 rh + rl) back to int8
    [N, K]: element (16 tile + g + 8 rl, 32 blk + 16 s + 8 rh + 2 t + e)."""
    x = q.reshape(N // 16, K // 32, 8, 4, 2, 2, 2, 2)  # tile, blk, g, t, s, rh, rl, e
    return x.permute(0, 6, 2, 1, 4, 5, 3, 7).reshape(N, K)


def rnd(*shape, seed=0, scale=1.0, dtype=bf16):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def close(a, b, what=""):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs()
    bad = (err > GEMM_ATOL + GEMM_RTOL * b.abs()).sum().item()
    assert bad == 0, f"{what}: {bad}/{a.numel()} mismatches, max err {err.max().item():.4g}"


def force_small(ops, m):
    ops.lib.b200mix_debug_w8_small_max(m)


@pytest.mark.parametrize("N,K", [(64, 128), (4608, 3584), (3584, 18944), (37888, 3584)])
@pytest.mark.parametrize("dtype", [torch.float32, bf16])
def test_quantize_matches_oracle_bit_for_bit(ops, N, K, dtype):
    g = torch.Generator().manual_seed(N + K)
    w = torch.randn(N, K, generator=g) * 0.02
    w[0] = 0.0                                                    # all-zero row: scale 0, q 0
    w[1] = torch.arange(K, dtype=torch.float32).remainder(255) - 127.0  # absmax 127: scale 1, integers
    w[2, :8] = torch.tensor([127.0, 0.5, -0.5, 1.5, -2.5, 0.49999997, -126.5, 3.5])  # ties at scale 1
    w[2, 8:] = 0.0
    w[3] = -w[3].abs()                                            # largest magnitude negative -> -127
    w = w.to(dtype)
    q_ref, s_ref = weight_quantize(w.float())
    wq = ops.quantize_w8(w.cuda(), None)
    torch.cuda.synchronize()
    assert torch.equal(wq.scale.cpu(), s_ref)
    q = unlayout(wq.q.cpu(), N, K)
    assert torch.equal(q, q_ref), (q != q_ref).nonzero()[:8]
    assert int(q_ref[3].min()) == -127


def _epilogue_ref(acc, epi, bias, res):
    if epi in ("swiglu", "geglu"):
        z = acc + bias
        return z[:, 0::2] * (F.silu(z[:, 1::2]) if epi == "swiglu" else F.gelu(z[:, 1::2]))
    if epi == "plain":
        return acc
    if epi == "bias+silu":
        return F.silu(acc + bias)
    if epi == "bias+res":
        return acc + bias + res.float()
    return acc + bias  # f32


def _run(ops, a, wq, epi, bias, res):
    kw = dict(plain={}, f32=dict(out_fp32=True), swiglu=dict(glu=2), geglu=dict(glu=1),
              **{"bias+silu": dict(act=1), "bias+res": dict(residual=res)})[epi]
    return ops.linear(a, wq, None if epi == "plain" else bias, **kw)


_weights = {}


def _weight(ops, N, K):
    """One quantized weight per shape for the whole module, with its fp32 dequantized form on the device."""
    if (N, K) not in _weights:
        _weights.clear()
        g = torch.Generator(device="cuda").manual_seed(1)
        wq = ops.quantize_w8(torch.randn(N, K, generator=g, device="cuda") * K ** -0.5,
                             torch.empty(N * K, device="cuda", dtype=bf16))
        _weights[(N, K)] = (wq, dequantize(unlayout(wq.q, N, K), wq.scale))
    return _weights[(N, K)]


def _refs(a, w_deq, epi, bias, res):
    """The fp32 reference of each path: the weight-streaming kernel multiplies by q and scales the fp32 sum; the large-M
    path runs the bf16 GEMM on bf16(q * scale), so its reference is the fp32 GEMM on that bf16 weight (as the bf16
    linear tests compare against the fp32 GEMM of their bf16 weight)."""
    return {small: _epilogue_ref(a.float() @ (w_deq if small else w_deq.to(bf16).float()).t(), epi, bias, res)
            for small in (True, False)}


SHAPES_7B = [(4608, 3584), (3584, 3584), (37888, 3584), (3584, 18944)]
SHAPES_TINY = [(512, 256), (256, 256), (1024, 256), (256, 512)]


@pytest.mark.parametrize("M", [1, 2, 3, 5, 8, 9, 16, 31, 32, 33, 63, 64, 65, 128, 300])
@pytest.mark.parametrize("N,K", SHAPES_TINY + SHAPES_7B)
def test_linear_w8_both_paths_match_oracle(ops, M, N, K):
    """Both paths forced on the same inputs, each against its fp32 reference; the epilogue varies with the shape (the decoder's: bias on q|k|v, residual
    on o / down, SwiGLU on gate|up)."""
    epi = {0: "bias+res", 1: "bias+res", 2: "swiglu", 3: "bias+res"}[(SHAPES_TINY + SHAPES_7B).index((N, K)) % 4]
    if (N, K) in ((512, 256), (4608, 3584)):
        epi = "f32"
    a = rnd(M, K, seed=M)
    wq, w_deq = _weight(ops, N, K)
    bias = rnd(N, seed=2, dtype=torch.float32)
    res = rnd(M, N, seed=3)
    refs = _refs(a, w_deq, epi, bias, res)
    for small_max in (1 << 30, 0):
        force_small(ops, small_max)
        try:
            out = _run(ops, a, wq, epi, bias, res)
        finally:
            force_small(ops, -1)
        close(out, refs[small_max > 0], f"w8 {'small' if small_max else 'large'} M{M} {N}x{K} {epi}")


@pytest.mark.parametrize("epi", ["plain", "bias+silu", "bias+res", "f32", "swiglu", "geglu"])
@pytest.mark.parametrize("M", [1, 5, 33, 300])
def test_linear_w8_epilogues(ops, epi, M):
    N, K = 1024, 512
    a, bias, res = rnd(M, K, seed=4), rnd(N, seed=5, dtype=torch.float32), rnd(M, N, seed=6)
    wq = ops.quantize_w8(rnd(N, K, seed=7, scale=K ** -0.5), torch.empty(N * K, device="cuda", dtype=bf16))
    refs = _refs(a, dequantize(unlayout(wq.q, N, K), wq.scale), epi, bias, res)
    for small_max in (1 << 30, 0):
        force_small(ops, small_max)
        try:
            out = _run(ops, a, wq, epi, bias, res)
        finally:
            force_small(ops, -1)
        assert out.dtype == (torch.float32 if epi == "f32" else bf16)
        close(out, refs[small_max > 0], f"w8 M{M} {epi} small_max={small_max}")


@pytest.mark.parametrize("M,N,K", [(1, 3584, 18944), (8, 4608, 3584), (20, 3584, 3584), (3, 512, 256), (64, 256, 512)])
def test_linear_w8_split_invariant_and_reproducible(ops, M, N, K):
    a, bias = rnd(M, K, seed=8), rnd(N, seed=9, dtype=torch.float32)
    wq = ops.quantize_w8(rnd(N, K, seed=10, scale=K ** -0.5), None)
    force_small(ops, 1 << 30)
    try:
        base = ops.linear(a, wq, bias, out_fp32=True)
        assert torch.equal(base, ops.linear(a, wq, bias, out_fp32=True))
        for splits in (1, 2, 3, 5, 8):
            ops.lib.b200mix_debug_skinny_splits(splits)
            try:
                out = ops.linear(a, wq, bias, out_fp32=True)
            finally:
                ops.lib.b200mix_debug_skinny_splits(0)
            assert torch.equal(out, base), (splits, (out - base).abs().max().item())
    finally:
        force_small(ops, -1)


def test_linear_w8_large_path_reproducible(ops):
    M, N, K = 300, 3584, 3584
    a = rnd(M, K, seed=11)
    wq = ops.quantize_w8(rnd(N, K, seed=12, scale=K ** -0.5), torch.empty(N * K, device="cuda", dtype=bf16))
    assert torch.equal(ops.linear(a, wq), ops.linear(a, wq))


def test_linear_w8_refusals(ops):
    from paddlemix_b200._lib import Epilogue, lib
    from paddlemix_b200.ops import _p, _stream, make_epilogue
    a = rnd(128, 1024, seed=13)
    buf = torch.zeros(1024 * 1024, device="cuda", dtype=torch.int8)
    scale = torch.ones(1024, device="cuda")
    c = torch.empty(128 * 1024, device="cuda", dtype=bf16)

    def call(M, N, K, e=None, ws=None, ws_bytes=0):
        return lib.b200mix_linear_w8(_p(a), 1024, _p(buf), _p(scale), _p(c), N, M, N, K,
                                     None if e is None else ctypes.byref(e), ws, ws_bytes, _stream())
    assert call(1, 64, 96) == ERR_INVALID          # K % 64 != 0
    assert call(1, 24, 128) == ERR_INVALID         # N % 16 != 0
    assert call(SMALL_MAX + 1, 64, 128) == ERR_INVALID  # no workspace above the crossover
    ws = torch.empty(64 * 128, device="cuda", dtype=bf16)
    assert call(SMALL_MAX + 1, 64, 128, ws=_p(ws), ws_bytes=64 * 128 * 2 - 2) == ERR_INVALID  # too small
    assert call(SMALL_MAX + 1, 64, 128, ws=_p(ws), ws_bytes=64 * 128 * 2) == 0
    assert call(SMALL_MAX, 64, 128) == 0
    row = torch.zeros(64, device="cuda")
    for e in (make_epilogue(row_add=row, ld_row=64, rows_per_group=1), make_epilogue(row_gate=row, ld_row=64),
              make_epilogue(out_scale=0.5), make_epilogue(residual_row_mod=4)):
        assert call(1, 64, 128, e) == ERR_UNSUPPORTED
    e = Epilogue()
    e.stats_out = buf.data_ptr()
    assert call(1, 64, 128, e) == ERR_UNSUPPORTED
    n = ctypes.c_int64(-1)
    assert lib.b200mix_linear_w8_workspace_size(SMALL_MAX, 4608, 3584, ctypes.byref(n)) == 0 and n.value == 0
    assert lib.b200mix_linear_w8_workspace_size(SMALL_MAX + 1, 4608, 3584, ctypes.byref(n)) == 0
    assert n.value == 4608 * 3584 * 2
    torch.cuda.synchronize()
    wq = ops.quantize_w8(rnd(64, 128, seed=14), None)
    with pytest.raises(ValueError, match="out_scale"):
        ops.linear(a[:1, :128], wq, out_scale=2.0)
    with pytest.raises(ValueError, match="row_add"):
        ops.linear(a[:1, :128], wq, row_add=row[None])
    with pytest.raises(ops._lib.B200MixError):
        ops.linear(a[:, :128], wq)  # M = 128 without a workspace
    with pytest.raises(ops._lib.B200MixError):
        ops.quantize_w8(rnd(24, 128, seed=15), None)


@pytest.mark.parametrize("M,kernels", [(8, 1), (128, 2)])
def test_linear_w8_counts_its_launches(ops, M, kernels):
    """ops.launches() (bench.py's gpu_launches) counts what an int8 linear starts: the weight-streaming kernel up to
    SMALL_MAX rows, the bf16 expansion and the GEMM above."""
    wq = ops.quantize_w8(rnd(256, 128, seed=30), torch.empty(256 * 128, device="cuda", dtype=bf16))
    a = rnd(M, 128, seed=31)
    ops.linear(a, wq)
    torch.cuda.synchronize()
    before = ops.launches()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.zeros(1, device="cuda")  # a torch kernel first: the trace can miss the first kernel of its window
        torch.cuda.synchronize()
        ops.linear(a, wq)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    seen = [n for n in names if "at::" not in n]
    assert ops.launches() - before == len(seen) == kernels, names


# ---- the decoder with quant_type="weight_only_int8" ------------------------------------------------------------------
def _padded(cfg, grid, n_text, seed=7):
    g = torch.Generator().manual_seed(seed)
    m2 = cfg["vision"]["spatial_merge_size"] ** 2
    T = sum(t * h * w for t, h, w in grid)
    pv = torch.randn(T, 3 * 2 * 14 * 14, generator=g)
    seqs = [[cfg["vision_start_token_id"]] + [cfg["image_token_id"]] * (t * h * w // m2) + [cfg["vision_end_token_id"]] +
            torch.randint(0, 1000, (nt,), generator=g).tolist() for (t, h, w), nt in zip(grid, n_text)]
    S = max(len(x) for x in seqs)
    ids, am = torch.zeros(len(seqs), S, dtype=torch.long), torch.zeros(len(seqs), S, dtype=torch.long)
    for i, x in enumerate(seqs):
        ids[i, S - len(x):], am[i, S - len(x):] = torch.tensor(x), 1
    return ids, am, pv


def _check(o, r, what):
    o, r = o.float().cpu(), r.float()
    cos = F.cosine_similarity(o.flatten().double(), r.flatten().double(), dim=0).item()
    err = (o - r).abs().max().item() / r.abs().max().item()
    assert cos >= 0.999 and err <= 0.04, (what, cos, err)


def _tiny_w8(seed):
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = O.QWEN2VL_CONFIGS["tiny"]
    P = O.init_qwen2vl_params(cfg, seed=seed)
    model = Qwen2VLForConditionalGeneration(dict(cfg, quant_type="weight_only_int8")).load_state_dict(P, device=0)
    return cfg, P, model


def test_qwen2vl_w8_prefill_and_decode_match_oracle_on_dequantized_weights():
    cfg, P, model = _tiny_w8(20)
    D = dequantize_decoder_params(cfg, P)
    grid = [[1, 8, 8], [1, 4, 8], [1, 8, 8]]
    ids, am, pv = _padded(cfg, grid, [30, 9, 60])
    model.cache_headroom = 4
    out = model(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    ref = O.qwen2vl_prefill(cfg, D, ids, pv, grid, attention_mask=am)
    keep = am.bool()
    _check(out.logits.cpu()[keep], ref[keep], "prefill")
    g = torch.Generator().manual_seed(21)
    for step in range(3):
        new = torch.randint(0, 1000, (ids.shape[0], 1), generator=g)
        o = model(input_ids=new, past_key_values=out.past_key_values, rope_deltas=out.rope_deltas, use_cache=True)
        ids, am = torch.cat([ids, new], 1), torch.cat([am, torch.ones_like(new)], 1)
        _check(o.logits[:, 0], O.qwen2vl_prefill(cfg, D, ids, pv, grid, attention_mask=am)[:, -1], f"decode {step}")


def test_qwen2vl_w8_graphed_step_equals_eager():
    from paddlemix_b200 import ops
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep
    cfg, _, model = _tiny_w8(22)
    grid = [[1, 8, 8], [1, 4, 8]]
    ids, am, pv = _padded(cfg, grid, [20, 9])
    B = ids.shape[0]
    model.cache_headroom = 8
    kw = dict(input_ids=ids, attention_mask=am, pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), use_cache=True)
    a, b = model(**kw), model(**kw)
    assert torch.equal(a.logits, b.logits)
    stepper = GraphedDecodeStep(model, b.past_key_values, b.rope_deltas)
    g = torch.Generator().manual_seed(23)
    for step in range(4):
        new = torch.randint(0, 1000, (B, 1), generator=g)
        n0 = ops.launches()
        eager = model(input_ids=new, past_key_values=a.past_key_values, rope_deltas=a.rope_deltas, use_cache=True).logits
        assert ops.launches() - n0 == stepper.launches_per_step
        assert torch.equal(eager[:, 0], stepper.step(new.reshape(-1))), step


def test_qwen2vl_w8_generate_strategies_return_bf16_shapes():
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg, P, model = _tiny_w8(24)
    ref = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    grid = [[1, 8, 8], [1, 4, 8]]
    ids, am, pv = _padded(cfg, grid, [12, 9])
    kw = dict(pixel_values=pv.cuda(), image_grid_thw=torch.tensor(grid), attention_mask=am, max_new_tokens=6)
    for extra in (dict(), dict(do_sample=True, top_k=20, generator=torch.Generator().manual_seed(3)),
                  dict(decode_strategy="beam_search", num_beams=3)):
        got = model.generate(ids, **kw, **extra)
        want = ref.generate(ids, **kw, **{k: (torch.Generator().manual_seed(3) if k == "generator" else v)
                                          for k, v in extra.items()})
        assert got.shape == want.shape and torch.equal(got[:, :ids.shape[1]], ids), extra


def test_llama_w8_prefill_matches_oracle_on_dequantized_weights():
    from paddlemix_b200.llava import LlamaForCausalLM
    cfg = dict(OL.LLAMA_CONFIGS["tiny"])
    P = OL.init_params(OL.llama_param_shapes(cfg), seed=3)
    model = LlamaForCausalLM(dict(cfg, quant_type="weight_only_int8")).load_state_dict(P, device=0)
    ids = torch.randint(0, cfg["vocab_size"], (2, 40), generator=torch.Generator().manual_seed(2))
    _check(model(input_ids=ids).logits, OL.llama_forward(cfg, dequantize_decoder_params(cfg, P, prefix="llama"), ids),
           "llama w8")


def test_w8_layer_weights_take_at_most_051_of_bf16_bytes():
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg, P, model = _tiny_w8(25)
    ref = Qwen2VLForConditionalGeneration(cfg).load_state_dict(P, device=0)
    names = ("qkv", "o", "gu", "down")
    w8 = sum(L[n].q.nbytes + L[n].scale.nbytes for L in model.decoder.layers for n in names)
    b16 = sum(L[n].nbytes for L in ref.decoder.layers for n in names)
    assert w8 <= 0.51 * b16, (w8, b16)
