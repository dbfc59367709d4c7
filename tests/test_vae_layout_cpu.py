"""oracle.vae.vae_decoder_layout, which the VAE production-geometry suite derives its call sites from, against the
decoder's parameter shapes: every site reads the parameters of its own shape, and every parameter is read by a site."""
import pytest

from oracle import vae as OV

def expected_shapes(s):
    """The parameters a site reads, with the shapes its op implies."""
    i, o = s["cin"], s["cout"]
    if s["op"] == "attention":
        return {f"{s['name']}.{n}.{k}": shp for n in ("to_q", "to_k", "to_v", "to_out.0")
                for k, shp in (("weight", (o, i)), ("bias", (o,)))}
    k = {"small_cin": 3, "conv3x3": 3, "up2x": 3, "shortcut": 1}.get(s["op"])
    if s["name"] == "post_quant_conv":
        k = 1
    w = (i,) if s["op"] == "groupnorm" else (o, i, k, k)
    return {s["name"] + ".weight": w, s["name"] + ".bias": (o,)}


@pytest.mark.parametrize("name", list(OV.VAE_CONFIGS))
def test_layout_matches_param_shapes(name):
    cfg = OV.VAE_CONFIGS[name]
    shapes = OV.vae_decoder_param_shapes(cfg)
    seen = {}
    for s in OV.vae_decoder_layout(cfg, 2, 16, 24):
        for k, shp in expected_shapes(s).items():
            assert k not in seen, f"{k} read by two sites"
            assert shapes.get(k) == shp, (k, shapes.get(k), shp)
            seen[k] = shp
    assert seen == shapes


def test_layout_geometry():
    """Spatial sizes and the tensor sizes the suite relies on: the SDXL decode at batch 8 reaches exactly 2^31 elements
    at up_blocks.2's upsampler output, Open-Sora's 64 frames at 512^2 reach 2^32."""
    cfg = OV.VAE_CONFIGS["sdxl_vae"]
    sites = OV.vae_decoder_layout(cfg, 8, 128, 128)
    assert [s["op"] for s in sites[:2]] == ["small_cin", "small_cin"]
    assert sites[-1]["name"] == "decoder.conv_out" and (sites[-1]["H"], sites[-1]["W"], sites[-1]["cout"]) == (1024, 1024, 3)
    att = next(s for s in sites if s["op"] == "attention")
    assert att["H"] * att["W"] == 16384 and att["cin"] == 512
    up = {s["name"]: s for s in sites if s["op"] == "up2x"}
    assert len(up) == 3
    u2 = up["decoder.up_blocks.2.upsamplers.0.conv"]
    assert u2["B"] * 4 * u2["H"] * u2["W"] * u2["cout"] == 2 ** 31
    r = {s["name"]: s for s in sites}
    assert r["decoder.up_blocks.3.resnets.0.norm1"]["cin"] == 256 and r["decoder.up_blocks.3.resnets.0.conv_shortcut"]["cout"] == 128
    u2 = next(s for s in OV.vae_decoder_layout(OV.VAE_CONFIGS["sd_vae"], 64, 64, 64) if s["name"] == u2["name"])
    assert u2["B"] * 4 * u2["H"] * u2["W"] * u2["cout"] == 2 ** 32
    bucket = OV.vae_decoder_layout(cfg, 3, 152, 104)
    assert next(s for s in bucket if s["op"] == "attention")["H"] * 104 == 15808
