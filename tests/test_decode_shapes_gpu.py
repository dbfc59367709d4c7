"""The decode step at the Qwen2-VL layer geometries generate() runs (7B: 28 query / 4 KV heads of 128, hidden 3584, MLP
18944, vocab 152064), each kernel against a plain high-precision evaluation of the same operation:

  a. the GQA-folded cache attention of decoder.decode_attention (head_dim 128 and 64) vs an fp64 softmax per unfolded
     head, with stale rows past kv_len and -inf key padding that masks whole key blocks;
  b. the fused RoPE / cache write (decode_rope_cache) vs rope_inplace (bit for bit) and an fp64 rotation;
  c. the embedding gather / image-token scatter on a 152064 x 3584 table;
  d. the decoder's five GEMMs with their epilogues at decode M (weight-streaming and tensor-core kernels);
  e. two layers at the 7B geometry end to end: eager and graphed decode steps up to a full cache vs the model's own
     prefill of the extended batch (and, marked slow, vs the fp32 host oracle).
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# (heads, kv_heads, head_dim): Qwen2-VL 7B (G = 7), 2B (G = 6), 72B (G = 8), no sharing (G = 1), the tiny config (D = 64)
GEOMETRIES = [(28, 4, 128), (12, 2, 128), (64, 8, 128), (4, 4, 128), (4, 2, 64)]
ATT_ATOL, ATT_RTOL = 1.5e-2, 2e-2  # as the other attention tests (test_ops_gpu.py)
GEMM_RTOL, GEMM_ATOL = 1.0e-2, 2e-2  # bf16 output of an fp32-accumulated dot product (test_ops_gpu.py)
COS_MIN, ERR_MAX = 0.999, 0.04  # end-to-end logits bar of the suite (test_baseline_parity_gpu.py)
STALE = 3.0e4  # cache rows at or past kv_len: large and finite, so any weight they get shows in the output


@pytest.fixture(scope="module")
def ops():
    from paddlemix_b200 import ops as _ops
    _ops.init(0)
    return _ops


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _qkv_rows(B, width, g, pad=24):
    """A [B, width] bf16 row view with a padded row stride (as a GEMM output inside a larger buffer), and its buffer."""
    buf = torch.randn(B, width + pad, generator=g, device="cuda").to(bf16)
    return buf[:, :width], buf


# ---------------------------------------------------------------------------------------------------------------------
# a. folded decode attention
# ---------------------------------------------------------------------------------------------------------------------
def _kv_lens_and_pads(B, max_len, salt):
    """Per-row key counts around the 64- and 128-key block edges, 640 and max_len (B = 1: max_len), and left-padding
    lengths of 0, 5 and whole blocks (64, 130)."""
    lens = [1, 63, 64, 65, 127, 128, 129, 640, max_len]
    pads = [0, 5, 64, 130]
    kv = [lens[(3 * b + salt) % len(lens)] for b in range(B)] if B > 1 else [max_len]
    # a padded prefix always leaves the row at least one visible key (the newest token is never padding)
    pad = [pads[(b + salt) % len(pads)] if pads[(b + salt) % len(pads)] < n else max(p for p in pads if p < n)
           for b, n in enumerate(kv)]
    return kv, pad


def _stale_cache(B, max_len, kvh, hd, kv, g):
    """[B, max_len, kvh, hd] bf16: randn below kv_len[b], +-STALE at and past it."""
    c = torch.randn(B, max_len, kvh, hd, generator=g, device="cuda")
    stale = torch.arange(max_len, device="cuda")[None, :] >= torch.tensor(kv, device="cuda")[:, None]
    c[stale] = STALE * torch.sign(c[stale] + 1e-3)
    return c.to(bf16)


def _ref_decode_attention(q, ck, cv, kv, bias, G):
    """fp64 softmax(q k^T / sqrt(hd) + bias) v over keys [0, kv_len) per sequence; query head h reads KV head h // G.
    q [B, heads, hd] -> [B, heads, hd] fp64."""
    hd = q.shape[-1]
    out = torch.empty(q.shape, dtype=torch.float64, device=q.device)
    for b, n in enumerate(kv):
        k = ck[b, :n].double().repeat_interleave(G, 1)  # [n, heads, hd]
        v = cv[b, :n].double().repeat_interleave(G, 1)
        s = torch.einsum("hd,nhd->hn", q[b].double(), k) / math.sqrt(hd)
        if bias is not None:
            s = s + bias[b, :n].double()[None]
        out[b] = torch.einsum("hn,nhd->hd", torch.softmax(s, -1), v)
    return out


def _close(a, b, atol, rtol, what):
    a, b = a.double(), b.double()
    err = (a - b).abs()
    bad = err > atol + rtol * b.abs()
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())}/{a.numel()} mismatches, max err {err.max().item():.4g}, "
                                 f"first at {tuple(bad.nonzero()[0].tolist())}")


@pytest.mark.parametrize("B", [1, 3, 32])
@pytest.mark.parametrize("masked", [False, True], ids=["no_bias", "left_pad"])
@pytest.mark.parametrize("heads,kv_heads,hd", GEOMETRIES)
def test_folded_decode_attention_vs_fp64(ops, heads, kv_heads, hd, masked, B):
    from paddlemix_b200.decoder import decode_attention
    G, qd = heads // kv_heads, heads * hd
    salt = GEOMETRIES.index((heads, kv_heads, hd)) + 2 * masked
    max_len = 701 + 53 * salt + B  # 700 .. 1100, not a multiple of any key block
    g = _gen(1000 + 17 * salt + B)
    kv, pad = _kv_lens_and_pads(B, max_len, salt)
    qkv, _ = _qkv_rows(B, (heads + 2 * kv_heads) * hd, g)
    ck, cv = _stale_cache(B, max_len, kv_heads, hd, kv, g), _stale_cache(B, max_len, kv_heads, hd, kv, g)
    kv_lens = torch.tensor(kv, dtype=torch.int32, device="cuda")
    bias = None
    if masked:
        bias = torch.zeros(B, max_len, device="cuda")
        for b, p in enumerate(pad):
            bias[b, :p] = float("-inf")
    # the output lands in a NaN-filled buffer with a padded row stride: every element of [B, qd] is written, nothing else
    big = torch.full((B + 2, qd + 40), float("nan"), device="cuda", dtype=bf16)
    out = big[1:B + 1, 16:16 + qd]
    got = decode_attention(qkv, ck, cv, heads, kv_heads, hd, kv_lens, bias, out=out)
    assert got.data_ptr() == out.data_ptr()
    assert torch.isfinite(out).all(), "unwritten or non-finite output"
    outside = torch.ones_like(big, dtype=torch.bool)
    outside[1:B + 1, 16:16 + qd] = False
    assert big[outside].isnan().all(), "wrote outside the output rows"

    q = qkv[:, :qd].unflatten(-1, (heads, hd))
    ref = _ref_decode_attention(q, ck, cv, kv, bias, G)
    what = f"heads {heads}/{kv_heads} hd {hd} B {B} kv {kv} pad {pad if masked else None}"
    _close(out.unflatten(-1, (heads, hd)), ref, ATT_ATOL, ATT_RTOL, "folded vs fp64, " + what)  # per unfolded head
    # the same inputs with every query head a head of its own (Sq = 1, Hq = heads)
    unfolded = ops.sdpa(q.unsqueeze(1), ck, cv, scale=hd ** -0.5, kv_lens=kv_lens,
                        attn_mask=None if bias is None else bias[:, None, None, :])
    _close(out.unflatten(-1, (heads, hd)), unfolded[:, 0].float(), ATT_ATOL, ATT_RTOL, "folded vs unfolded, " + what)


# ---------------------------------------------------------------------------------------------------------------------
# b. decode_rope_cache
# ---------------------------------------------------------------------------------------------------------------------
def _bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (8 significant bits)."""
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), e - 8)


@pytest.mark.parametrize("table", ["rope", "general"])
@pytest.mark.parametrize("B", [1, 3, 32])
@pytest.mark.parametrize("heads,kv_heads,hd", GEOMETRIES)
def test_decode_rope_cache(ops, heads, kv_heads, hd, B, table):
    """table "rope": decoder.rope_cos_sin at a position per row up to 32k (its two halves are equal); "general": an
    independent angle per column, which the kernels' [B, head_dim] tables allow."""
    from paddlemix_b200.decoder import rope_cos_sin
    qd, kvd = heads * hd, kv_heads * hd
    g = _gen(2000 + GEOMETRIES.index((heads, kv_heads, hd)) + B)
    qkv, buf = _qkv_rows(B, qd + 2 * kvd, g)
    x0 = buf.clone()
    n_rows = 3 * 257  # flattened cache rows (3 sequences of 257 positions); B of them are written
    inner = torch.randperm(n_rows - 2, generator=g, device="cuda")[:max(B - 2, 0)] + 1
    rows = torch.cat([torch.tensor([0], device="cuda")[:B - 1], inner, torch.tensor([n_rows - 1], device="cuda")])
    assert rows.unique().numel() == B  # distinct, the last row always, row 0 when B > 1
    if table == "rope":
        pos = torch.randint(0, 32768, (B,), generator=g, device="cuda")
        pos[0] = 32767
        cos_t, sin_t = rope_cos_sin(1e6, hd, 32768)
        cos, sin = cos_t.cuda()[pos].contiguous(), sin_t.cuda()[pos].contiguous()
    else:
        ang = torch.rand(B, hd, generator=g, device="cuda") * (2 * math.pi)
        cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    sentinel = -1234.0
    ck = torch.full((n_rows, kvd), sentinel, device="cuda", dtype=bf16)
    cv = torch.full((n_rows, kvd), sentinel, device="cuda", dtype=bf16)

    ops.decode_rope_cache(qkv, heads, kv_heads, hd, cos, sin, rows, ck, cv)

    q_rope = x0[:, :qd].clone().unflatten(-1, (heads, hd))
    k_rope = x0[:, qd:qd + kvd].clone().unflatten(-1, (kv_heads, hd))
    ops.rope_inplace(q_rope, cos, sin)
    ops.rope_inplace(k_rope, cos, sin)
    want = x0.clone()
    want[:, :qd] = q_rope.flatten(1)
    # q rotated in place bit for bit as rope_inplace; the k / v part and the row padding untouched
    assert torch.equal(buf, want), f"qkv rows: {int((buf != want).sum())} elements differ"
    want_k = torch.full_like(ck, sentinel)
    want_v = torch.full_like(cv, sentinel)
    want_k[rows] = k_rope.flatten(1)
    want_v[rows] = x0[:, qd + kvd:qd + 2 * kvd]
    assert torch.equal(ck, want_k), f"k cache: {int((ck != want_k).sum())} elements differ"
    assert torch.equal(cv, want_v), f"v cache: {int((cv != want_v).sum())} elements differ"

    # and within one bf16 ulp of the rotation in fp64 (on the same fp32 cos / sin), plus the fp32 rounding of the two
    # products it is the sum of (which dominates only where they cancel)
    x = x0[:, :qd].unflatten(-1, (heads, hd)).double()
    rot = torch.cat([-x[..., hd // 2:], x[..., :hd // 2]], -1)
    t1, t2 = x * cos.double()[:, None], rot * sin.double()[:, None]
    ref = t1 + t2
    err = (buf[:, :qd].unflatten(-1, (heads, hd)).double() - ref).abs()
    tol = _bf16_ulp(ref) + 2.0 ** -23 * (t1.abs() + t2.abs())
    assert bool((err <= tol).all()), f"q rope: max err {err.max().item():.3g} exceeds one bf16 ulp"


# ---------------------------------------------------------------------------------------------------------------------
# c. gather_rows / scatter_rows
# ---------------------------------------------------------------------------------------------------------------------
def test_gather_scatter_rows_vocab_table(ops):
    V, D, n = 152064, 3584, 3000  # n * D / 8 vectors: several rounds of the grid-stride loop
    g = _gen(3000)
    table = torch.randn(V, D, generator=g, device="cuda").to(bf16)
    ids = torch.randint(0, V, (n,), generator=g, device="cuda")
    ids[:4] = torch.tensor([0, V - 1, 0, V - 1])
    ids[-100:] = ids[100:200]  # repeats
    got = ops.gather_rows(table, ids)
    assert got.shape == (n, D) and torch.equal(got, table[ids])

    R, sentinel = 5000, 777.0
    dst = torch.full((R, D), sentinel, device="cuda", dtype=bf16)
    idx = torch.cat([torch.tensor([R - 1, 0], device="cuda"), torch.randperm(R - 2, generator=g, device="cuda")[:n - 2] + 1])
    src = torch.randn(n, D, generator=g, device="cuda").to(bf16)
    ops.scatter_rows(src, idx, dst)
    want = torch.full_like(dst, sentinel)
    want[idx] = src
    assert torch.equal(dst, want), f"scatter: {int((dst != want).any(1).sum())} rows differ"


# ---------------------------------------------------------------------------------------------------------------------
# d. the decoder's GEMMs at decode M
# ---------------------------------------------------------------------------------------------------------------------
H7, I7, V7, KV7 = 3584, 18944, 152064, 4 * 128
M_MAX = 32


@pytest.fixture(scope="module")
def decoder_gemms():
    """The five 7B GEMMs as CausalDecoder runs them (weight [N, K] bf16, epilogue), drawn once per module with M_MAX
    input rows and the fp32 reference of every row: a row's result does not depend on M."""
    from paddlemix_b200._lib import GLU_SWIGLU
    g = _gen(4000)

    def w(N, K):
        return ((torch.rand(N, K, generator=g, device="cuda") * 2 - 1) * K ** -0.5).to(bf16)

    cases = {}
    for name, N, K in (("qkv", H7 + 2 * KV7, H7), ("o", H7, H7), ("gate_up", 2 * I7, H7), ("down", H7, I7),
                       ("lm_head", V7, H7)):
        wt = w(N, K)
        a = torch.randn(M_MAX, K, generator=g, device="cuda").to(bf16)
        acc = a.float() @ wt.float().t()
        kw, extra = {}, {}
        if name == "qkv":
            kw["bias"] = 0.05 * torch.randn(N, generator=g, device="cuda")
            ref = acc + kw["bias"]
        elif name in ("o", "down"):
            extra["residual"] = torch.randn(M_MAX, N, generator=g, device="cuda").to(bf16)
            ref = acc + extra["residual"].float()
        elif name == "gate_up":
            kw["glu"] = GLU_SWIGLU
            ref = acc[:, 0::2] * F.silu(acc[:, 1::2])  # interleaved rows: 2j = up (value), 2j + 1 = gate
        else:
            kw["out_fp32"] = True
            ref = acc
        cases[name] = (a, wt, kw, extra, ref)
        del acc
    return cases


@pytest.mark.parametrize("M", [1, 3, 8, 9, 32])
@pytest.mark.parametrize("name", ["qkv", "o", "gate_up", "down", "lm_head"])
def test_decoder_gemm_at_decode_m(ops, decoder_gemms, name, M):
    a, wt, kw, extra, ref = decoder_gemms[name]
    out = ops.linear(a[:M], wt, **kw, **{k: v[:M] for k, v in extra.items()})
    assert out.dtype == (torch.float32 if kw.get("out_fp32") else bf16) and out.shape == ref[:M].shape
    _close(out, ref[:M], GEMM_ATOL, GEMM_RTOL, f"{name} {tuple(wt.shape)} M {M}")


# ---------------------------------------------------------------------------------------------------------------------
# e. two layers at the 7B geometry, eager and graphed decode up to a full cache
# ---------------------------------------------------------------------------------------------------------------------
N_EAGER, N_GRAPHED = 3, 4


def _cfg_7b_two_layers():
    from oracle import qwen2vl as O
    cfg = dict(O.QWEN2VL_CONFIGS["qwen2vl_7b"], num_hidden_layers=2)
    cfg["vision"] = dict(cfg["vision"], depth=1)
    return cfg


@pytest.fixture(scope="module")
def qwen7b_two_layers():
    """(cfg, bf16 state dict on the device, {quant_type: model}) -- both models load the same synthetic weights."""
    from paddlemix_b200.modeling import synthetic_state_dict
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    cfg = _cfg_7b_two_layers()
    shapes = Qwen2VLForConditionalGeneration(cfg).state_dict_shapes()
    P = synthetic_state_dict(shapes, 5, 0, lambda name, shp, randn: 0.5 * randn(shp)
                             if name == "model.embed_tokens.weight" else None)
    models = {q: Qwen2VLForConditionalGeneration(dict(cfg, quant_type=q)).load_state_dict(P, device=0)
              for q in (None, "weight_only_int8")}
    return cfg, P, models


def _prompt(B, S, pads, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 151643, (B, S), generator=g)
    am = torch.ones(B, S, dtype=torch.long)
    for b, p in enumerate(pads):
        ids[b, :p], am[b, :p] = 0, 0
    return ids, (am if any(pads) else None)


def _decode_run(model, ids, am):
    """Prefill two caches of max_len = S + N_EAGER + N_GRAPHED; run N_EAGER eager steps on both, then eager steps on one
    and graphed steps on the other until both are full. Returns (new tokens [B, n], eager logits, graphed logits) with
    logits on the host, one [B, vocab] per step (graphed: None for the eager-only steps)."""
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep
    B, S = ids.shape
    n = N_EAGER + N_GRAPHED
    model.cache_headroom = n
    a = model(input_ids=ids, attention_mask=am, use_cache=True)
    b = model(input_ids=ids, attention_mask=am, use_cache=True)
    assert a.past_key_values.max_len == S + n
    new = torch.randint(0, 151643, (B, n), generator=torch.Generator().manual_seed(S))
    eager, graphed, stepper = [], [], None
    for t in range(n):
        tok = new[:, t:t + 1]
        e = model(input_ids=tok, past_key_values=a.past_key_values, rope_deltas=a.rope_deltas, use_cache=True).logits[:, 0]
        eager.append(e.cpu())
        if t < N_EAGER:
            model(input_ids=tok, past_key_values=b.past_key_values, rope_deltas=b.rope_deltas, use_cache=True)
            graphed.append(None)
            continue
        if stepper is None:
            stepper = GraphedDecodeStep(model, b.past_key_values, b.rope_deltas)
        graphed.append(stepper.step(tok.reshape(-1)).cpu())
    for cache in (a.past_key_values, b.past_key_values):
        assert cache.length == cache.max_len  # the last step wrote the last cache row (kv_len == max_len)
    with pytest.raises(ValueError, match="full"):
        stepper.step(new[:, 0])
    with pytest.raises(ValueError, match="full"):
        model(input_ids=new[:, :1], past_key_values=a.past_key_values, rope_deltas=a.rope_deltas, use_cache=True)
    return new, eager, graphed


def _assert_rows_close(got, ref, what):
    """Per sequence: cosine >= COS_MIN and max |err| <= ERR_MAX * max |ref| (the suite's end-to-end bar)."""
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape and torch.isfinite(got).all(), what
    cos = F.cosine_similarity(got, ref, dim=-1)
    err = (got - ref).abs().amax(-1) / ref.abs().amax(-1)
    assert bool((cos >= COS_MIN).all() and (err <= ERR_MAX).all()), (what, cos.tolist(), err.tolist())


# B = 3: left padding of 0 / 70 / 131 tokens (whole 64-key blocks masked), decode crossing the key block at 192;
# B = 32: unpadded, every decode GEMM at M = 32
E2E_BATCHES = {3: (190, (0, 70, 131)), 32: (60, (0,) * 32)}


@pytest.mark.parametrize("B", sorted(E2E_BATCHES))
@pytest.mark.parametrize("quant", [None, "weight_only_int8"], ids=["bf16", "w8"])
def test_7b_geometry_decode_vs_prefill(qwen7b_two_layers, quant, B):
    """Every decode step's logits against the model's own prefill of the extended (still padded) batch at its last
    position: an independent kernel path (rope_inplace, masked multi-row attention, M = B * S GEMMs). Graphed steps
    equal eager steps bit for bit."""
    cfg, _, models = qwen7b_two_layers
    model = models[quant]
    S, pads = E2E_BATCHES[B]
    ids, am = _prompt(B, S, pads, seed=B)
    new, eager, graphed = _decode_run(model, ids, am)
    for t in range(new.shape[1]):
        ext = torch.cat([ids, new[:, :t + 1]], 1)
        ext_am = None if am is None else torch.cat([am, torch.ones(B, t + 1, dtype=torch.long)], 1)
        ref = model(input_ids=ext, attention_mask=ext_am).logits[:, -1].cpu()
        _assert_rows_close(eager[t], ref, f"{quant} B {B} step {t} (kv_len {S + t + 1})")
        if graphed[t] is not None:
            assert torch.equal(graphed[t], eager[t]), f"{quant} B {B} step {t}: graphed != eager"


@pytest.mark.slow
def test_7b_geometry_decode_vs_oracle(qwen7b_two_layers):
    """The bf16, B = 3 padded run against the fp32 host oracle: one prefill of the final extended batch gives every
    step's reference at its position (causal attention: position S + t sees the same keys as decode step t)."""
    from oracle import qwen2vl as O
    cfg, P, models = qwen7b_two_layers
    S, pads = E2E_BATCHES[3]
    ids, am = _prompt(3, S, pads, seed=3)
    new, eager, graphed = _decode_run(models[None], ids, am)
    ext = torch.cat([ids, new], 1)
    ext_am = torch.cat([am, torch.ones_like(new)], 1)
    Ph = {k: v.float().cpu() for k, v in P.items() if not k.startswith("visual.")}
    with torch.no_grad():
        ref = O.qwen2vl_prefill(cfg, Ph, ext, None, None, attention_mask=ext_am)
    for t in (0, new.shape[1] - 1):
        got = eager[t] if graphed[t] is None else graphed[t]
        _assert_rows_close(got, ref[:, S + t], f"oracle step {t} ({'eager' if graphed[t] is None else 'graphed'})")
