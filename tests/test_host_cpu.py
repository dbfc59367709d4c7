"""CPU-side checks: the C-ABI library loads and exports every symbol include/b200mix.h declares, refuses to run
without a GPU (no fallback), the host mirror builds the same structure as the oracle, and the multi-rank plumbing
(batch sharding + all_gather of finished latents) works under gloo with world_size 2."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from paddlemix_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "b200mix.h")).read()
    declared = set(re.findall(r"\b(b200mix_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"b200mix_epilogue", "b200mix_status"}
    assert len(declared) >= 20
    for name in sorted(declared):
        assert hasattr(_lib.lib, name), f"{name} declared in include/b200mix.h but not exported"
    assert set(_lib.SIGNATURES) | set(_lib.STRING_GETTERS) == declared


def test_no_cpu_fallback():
    from paddlemix_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    rc = _lib.lib.b200mix_init(0)
    assert rc == -3
    assert b"no CPU fallback" in _lib.lib.b200mix_last_error()
    from paddlemix_b200 import ops
    with pytest.raises(_lib.B200MixError):
        ops.linear(torch.zeros(8, 64, dtype=torch.bfloat16), torch.zeros(8, 64, dtype=torch.bfloat16))


def test_unet_structure_matches_oracle():
    from oracle import unet as O
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    for name in ("sd15", "sdxl", "tiny_sd", "tiny_xl"):
        cfg = O.UNET_CONFIGS[name]
        keys = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels",
                "layers_per_block", "cross_attention_dim", "transformer_layers_per_block", "attention_head_dim",
                "use_linear_projection", "addition_embed_type", "addition_time_embed_dim",
                "projection_class_embeddings_input_dim")
        m = UNet2DConditionModel(**{k: cfg[k] for k in keys})
        shapes = O.unet_param_shapes(cfg)
        assert m.state_dict_shapes() == shapes  # same parameter names and (Paddle-layout) shapes as the oracle
        names = {r.name for r in m.resnets} | {t.name for t in m.transformers}
        for r in m.resnets:
            assert shapes[r.name + ".conv1.weight"] == (r.cout, r.cin, 3, 3)
            assert ((r.name + ".conv_shortcut.weight") in shapes) == (r.shortcut is not None)
        n_attn = sum(2 * len(t.blocks) for t in m.transformers)
        assert len(m.attn_processors) == n_attn
        assert n_attn == sum(1 for k in shapes if k.endswith(".to_q.weight"))
        assert len(names) == len(m.resnets) + len(m.transformers)
    assert len(UNet2DConditionModel(**{k: O.UNET_CONFIGS["sdxl"][k] for k in keys}).attn_processors) == 140


def test_sd3_structure_matches_oracle():
    from oracle import sd3 as O3
    from paddlemix_b200.ppdiffusers.transformer_sd3 import SD3Transformer2DModel
    for name in ("sd3_medium", "tiny"):
        cfg = O3.SD3_CONFIGS[name]
        assert SD3Transformer2DModel(**cfg).state_dict_shapes() == O3.sd3_param_shapes(cfg)
    assert abs(O3.sd3_flops(O3.SD3_CONFIGS["sd3_medium"], 1, 128, 128, 154) / 1e12 - 8.437) < 5e-3


def test_qwen2vl_structure_and_rope_index_match_oracle():
    from oracle import qwen2vl as OQ
    from paddlemix_b200.qwen2_vl import Qwen2VLForConditionalGeneration
    for name in ("qwen2vl_7b", "tiny"):
        cfg = OQ.QWEN2VL_CONFIGS[name]
        assert Qwen2VLForConditionalGeneration(cfg).state_dict_shapes() == OQ.qwen2vl_param_shapes(cfg)
    cfg = OQ.QWEN2VL_CONFIGS["qwen2vl_7b"]
    m = Qwen2VLForConditionalGeneration(cfg)
    g = torch.Generator().manual_seed(0)
    grid = [[1, 32, 32]] * 2  # BASELINE config C4: 448x448 image -> 1024 patches -> 256 merged tokens + 510 text
    rows = [[cfg["vision_start_token_id"]] + [cfg["image_token_id"]] * 256 + [cfg["vision_end_token_id"]] +
            torch.randint(0, 151643, (510,), generator=g).tolist() for _ in range(2)]
    ids = torch.tensor(rows)
    po, do = OQ.get_rope_index(cfg, ids, grid)
    pm, dm = m.get_rope_index(ids, torch.tensor(grid))
    assert ids.shape == (2, 768) and torch.equal(po, pm) and torch.equal(do, dm)
    assert torch.equal(m.rot_pos_emb(grid), OQ.rot_pos_emb(cfg, grid))


def test_llama_structure_matches_oracle():
    from oracle import llama as OL
    from paddlemix_b200.llava import LlamaForCausalLM
    for name in ("tiny", "vicuna_7b"):
        cfg = OL.LLAMA_CONFIGS[name]
        assert LlamaForCausalLM(cfg).state_dict_shapes() == OL.llama_param_shapes(cfg)


def test_graphed_decode_step_needs_room_for_its_warmup():
    """The warm-up steps write cache rows length .. length + warmup - 1: a cache without that room is refused before
    any device work (the stand-in cache has no tensors and the model no weights, so nothing could be launched)."""
    from types import SimpleNamespace

    from oracle import qwen2vl as OQ
    from paddlemix_b200.qwen2_vl import GraphedDecodeStep, Qwen2VLForConditionalGeneration
    model = Qwen2VLForConditionalGeneration(OQ.QWEN2VL_CONFIGS["tiny"])
    for length, max_len, warmup in ((9, 10, 2), (10, 10, 2), (10, 10, 1), (3, 5, 3)):
        cache = SimpleNamespace(length=length, max_len=max_len, batch=2, key_bias=None, k=None, v=None)
        with pytest.raises(ValueError, match="warm-up"):
            GraphedDecodeStep(model, cache, None, warmup=warmup)


def test_stdit2_structure_matches_oracle():
    from oracle import stdit2 as OS2
    from paddlemix_b200.opensora import STDiT2
    for name in ("stdit2_xl", "tiny"):
        cfg = OS2.STDIT2_CONFIGS[name]
        assert STDiT2(cfg).state_dict_shapes() == OS2.stdit2_param_shapes(cfg)
    assert abs(OS2.stdit2_flops(OS2.STDIT2_CONFIGS["stdit2_xl"], 1, 16, 1024, 120) / 1e12 - 24.4) < 0.1


def test_config_errors_mirror_reference():
    from paddlemix_b200.ppdiffusers.unet_2d_condition import UNet2DConditionModel
    with pytest.raises(ValueError, match="same number of `down_block_types`"):
        UNet2DConditionModel(down_block_types=("DownBlock2D",), up_block_types=("UpBlock2D", "UpBlock2D"), block_out_channels=(64,))
    with pytest.raises(ValueError, match="num_attention_heads"):
        UNet2DConditionModel(num_attention_heads=8)
    m = UNet2DConditionModel()
    assert m.config.in_channels == 4 and m.in_channels == 4 and m.dtype == torch.bfloat16
    with pytest.raises(Exception):
        m.config.in_channels = 3
    with pytest.raises(RuntimeError):
        m.forward(torch.zeros(1, 4, 8, 8), 1, torch.zeros(1, 77, 1280))
    # options outside the hot path are refused unless they sit at the reference's own default; True == 1.0 / 0 == False
    # style coincidences must not slip through (each option is compared with ITS default, by type and value)
    for kw in (dict(dual_cross_attention=True), dict(resnet_skip_time_act=True), dict(class_embeddings_concat=True),
               dict(class_embed_type="timestep"), dict(conv_in_kernel=5), dict(conv_in_kernel=3.0),
               dict(time_embedding_type="fourier"), dict(attention_type="gated"), dict(not_a_reference_option=None)):
        with pytest.raises(NotImplementedError):
            UNet2DConditionModel(**kw)
    UNet2DConditionModel(dual_cross_attention=False, conv_in_kernel=3, upcast_attention=True, class_embed_type=None,
                         _class_name="UNet2DConditionModel")


def test_flops_match_survey():
    from oracle import unet as O
    assert abs(O.unet_flops(O.UNET_CONFIGS["sdxl"], 1, 128, 128, 77) / 1e12 - 6.761) < 5e-3
    assert abs(O.unet_flops(O.UNET_CONFIGS["sd15"], 1, 64, 64, 77) / 1e12 - 0.803) < 5e-3


def test_oracle_self_consistency():
    # ModelTesterMixin-style properties on the reference's own tiny config (test_models_unet_2d_condition.py:181-194)
    from oracle import unet as O
    cfg = O.UNET_CONFIGS["ref_tiny"]
    P = O.init_params(O.unet_param_shapes(cfg))
    g = torch.Generator().manual_seed(0)
    x, ctx = torch.randn(4, 4, 32, 32, generator=g), torch.randn(4, 4, 32, generator=g)
    y = O.unet_forward(cfg, P, x, 10, ctx)
    assert y.shape == x.shape and torch.equal(y, O.unet_forward(cfg, P, x, 10, ctx))
    one = O.unet_forward(cfg, P, x[1:2], torch.tensor([10]), ctx[1:2])
    assert torch.allclose(one, y[1:2], atol=1e-4)

    def sdpa_proc(x, c, P, p, heads, mask):  # processor-swap equivalence (test_modeling_common.py:197-256)
        c = x if c is None else c
        q, k, v = O.linear(x, P, p + ".to_q"), O.linear(c, P, p + ".to_k"), O.linear(c, P, p + ".to_v")
        B, S, C = q.shape
        sp = lambda t: t.reshape(B, -1, heads, C // heads).transpose(1, 2)
        o = torch.nn.functional.scaled_dot_product_attention(sp(q), sp(k), sp(v)).transpose(1, 2).reshape(B, S, C)
        return O.linear(o, P, p + ".to_out.0")
    y2 = O.unet_forward(cfg, P, x, 10, ctx, processor=sdpa_proc)
    assert (y - y2).abs().max() < 1e-3


WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from paddlemix_b200.ppdiffusers.pipelines import all_gather_latents, shard_batch
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
full = torch.arange(8 * 4 * 2 * 2, dtype=torch.float32).reshape(8, 4, 2, 2)
lo, hi = shard_batch(8, rank, 2)
mine = full[lo:hi] * 2.0            # "denoise" the local shard
out = all_gather_latents(mine)
assert out.shape == full.shape and torch.equal(out, full * 2.0), rank
assert shard_batch(5, 0, 2) == (0, 3) and shard_batch(5, 1, 2) == (3, 5)
dist.destroy_process_group()
print("ok", rank)
'''


def test_data_parallel_plumbing_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    port = str(29500 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for r in range(2)]
    for p in procs:
        out, _ = p.communicate(timeout=120)
        assert p.returncode == 0, out.decode()


def test_fold_layernorm_into_linear_algebra():
    """The load-time fold behind b200mix_epilogue.ln_stats: Linear(LayerNorm(h)) == rstd * (h W'^T - mean * colsum) + bias'
    (BasicTransformerBlock norm1/2/3 -> to_q|k|v / to_q / GEGLU proj, attention.py:352-489). fp64 on the CPU; the only
    difference left is the bf16 rounding of W' = W * gamma."""
    import torch
    import torch.nn.functional as F

    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(0)
    M, K, N = 37, 96, 40
    h = (torch.randn(M, K, generator=g) * 2 + 0.7).to(torch.bfloat16).double()
    w, b = torch.randn(N, K, generator=g) * K ** -0.5, torch.randn(N, generator=g)
    gamma, beta = 1 + 0.3 * torch.randn(K, generator=g), 0.2 * torch.randn(K, generator=g)
    w2, colsum, b2 = ops.fold_layernorm_into_linear(w, gamma, beta, b)
    assert w2.dtype == torch.bfloat16 and torch.equal(colsum, w2.float().sum(1))
    mean, var = h.mean(1, keepdim=True), h.var(1, unbiased=False, keepdim=True)
    rstd = torch.rsqrt(var + 1e-5)
    out = rstd * (h @ w2.double().t() - mean * colsum.double()[None]) + b2.double()[None]
    ref = F.linear(F.layer_norm(h, (K,), gamma.double(), beta.double(), 1e-5), w.double(), b.double())
    assert (out - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
    # with unrounded folded weights the identity is exact
    w2x = w.double() * gamma.double()[None]
    outx = rstd * (h @ w2x.t() - mean * w2x.sum(1)[None]) + (b.double() + w.double() @ beta.double())[None]
    assert (outx - ref).abs().max().item() < 1e-9
    # fixed-point row totals (2^24) reproduce mean / rstd the way the consuming epilogue rebuilds them
    tab = torch.stack([(h.sum(1) * ops.RowStats.SCALE).round(), ((h * h).sum(1) * ops.RowStats.SCALE).round()], 1).to(torch.int64)
    m2, r2 = ops.RowStats(tab, K).mean_rstd(1e-5)
    assert (m2.double() - mean[:, 0]).abs().max().item() < 1e-5 and (r2.double() / rstd[:, 0] - 1).abs().max().item() < 1e-4


def test_fold_upsample_conv_weight_algebra():
    """b200mix_conv3x3_up2x's per-parity 2x2 filters == F.interpolate(scale 2, nearest) + conv3x3 (Upsample2D,
    resnet.py:169-218), including the zero padding at every border."""
    import torch
    import torch.nn.functional as F

    from paddlemix_b200 import ops
    g = torch.Generator().manual_seed(1)
    O, I, H, W = 6, 5, 4, 7
    w = torch.randn(O, 3, 3, I, generator=g).to(torch.bfloat16).float()
    w4 = ops.fold_upsample_conv_weight(w).float().reshape(O, 2, 2, 2, 2, I)
    x = torch.randn(2, I, H, W, generator=g)
    ref = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w.permute(0, 3, 1, 2), padding=1)
    xp = F.pad(x, (1, 1, 1, 1))
    out = torch.zeros_like(ref)
    for py in range(2):
        for px in range(2):
            acc = 0
            for a in range(2):
                for b in range(2):
                    dy, dx = a - 1 + py, b - 1 + px  # the tap table of b200mix_conv3x3_up2x (csrc/gemm.cu)
                    acc = acc + torch.einsum("bchw,oc->bohw", xp[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W], w4[:, py, px, a, b])
            out[:, :, py::2, px::2] = acc
    assert (out - ref).abs().max().item() < 2e-2 * ref.abs().max().item()  # bf16 rounding of the summed taps only


def test_streamk_schedule_covers_every_k_block_once():
    """Python mirror of SegIter (csrc/gemm.cu): the stream-K head + round-robin rest visits every (tile, k-block) exactly
    once, every cluster gets the same number of k-blocks (+-1), a split tile has exactly one head piece (last piece of
    cluster c) and one tail piece (first piece of cluster c + 1)."""
    import random

    def segs(sk_tiles, total, kblocks, c, nc):
        units = sk_tiles * kblocks
        u, u1, out = c * units // nc, (c + 1) * units // nc, []
        while u < u1:
            st = u // kblocks
            kb0 = u - st * kblocks
            kb1 = min(kblocks, kb0 + (u1 - u))
            u += kb1 - kb0
            out.append((st, kb0, kb1))
        out += [(st, 0, kblocks) for st in range(sk_tiles + c, total, nc)]
        return out

    rnd = random.Random(0)
    checked = 0
    while checked < 300:
        nc, total, kb = rnd.randint(1, 74), rnd.randint(2, 1500), rnd.randint(8, 400)
        if total <= nc or total % nc == 0:
            continue
        checked += 1
        sk = nc + total % nc
        allsegs = [segs(sk, total, kb, c, nc) for c in range(nc)]
        seen = set()
        for c, ss in enumerate(allsegs):
            for i, (st, a, b) in enumerate(ss):
                assert a < b
                if a > 0:  # tail piece
                    assert i == 0 and b == kb
                    assert [s for s in allsegs[c - 1] if s[0] == st] == [(st, 0, a)]
                elif b < kb:  # head piece
                    assert allsegs[c + 1][0] == (st, b, kb)
                    assert all(s[1] == 0 and s[2] == kb for s in ss[i + 1:])
                for k in range(a, b):
                    assert (st, k) not in seen
                    seen.add((st, k))
        assert len(seen) == total * kb
        lens = [sum(b - a for _, a, b in ss) for ss in allsegs]
        assert max(lens) - min(lens) <= 1


def test_epilogue_struct_layout_matches_header(tmp_path):
    """The ctypes mirror of b200mix_epilogue (paddlemix_b200/_lib.py) against what a C compiler makes of include/b200mix.h:
    same size, same offset for every field (a silent mismatch would shift every epilogue pointer)."""
    import ctypes
    import os
    import subprocess

    from paddlemix_b200._lib import Epilogue
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields = [f[0] for f in Epilogue._fields_]
    src = tmp_path / "layout.c"
    lines = "".join(f'  printf("{f} %zu\\n", offsetof(b200mix_epilogue, {f}));\n' for f in fields)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200mix.h"\nint main(void) {\n'
                   '  printf("sizeof %zu\\n", sizeof(b200mix_epilogue));\n' + lines + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["sizeof"]) == ctypes.sizeof(Epilogue)
    for f in fields:
        assert int(out[f]) == getattr(Epilogue, f).offset, f
