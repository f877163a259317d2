"""CPU: the launches each conv layer expands into, recorded by the host-only twins of dmd_conv_layer_fprop / _dgrad / _wgrad.
Those twins run the executors' own expansions (the K-split chunks, split-fp16 passes, backward-data chunks and weight-gradient
blocks of every plan and of the actor-critic's immediate mode) on stand-in pointers, so these checks need no GPU:

- each layer gets the chunking, split-fp16 mode and backward-data chunk width that the layer walker's rules give;
- every stored input channel of every source is read by exactly one chunk (per pass), at its own PLC16 plane;
- only the first launch carries the bias and the caller's residual, every later one accumulates onto the output, and only the
  last carries the statistics; three-pass chunks run hi/hi, lo/hi, hi/lo with the low-part pack on the third pass only;
- backward-data chunk j reads the gradient from plane j * widthT / 8, and every chunk after the first accumulates;
- the weight-gradient blocks tile [0, Cout) x [ci_off, ci_off + Cin) exactly once, padding channels excluded.

tests/test_gpu_conv_layers.py runs the same layers on the GPU against float64."""
import pytest

from diamond_b200 import _lib, ops

# name -> the layer walker's arguments (cout, cin_real, taps, c0_real, c0_store, c1, split, dgrad), the conv's stride, and the
# expansion the walker's rules give: K-split chunks (stored channels each), split-fp16 mode, backward-data chunk width, launches
LAYERS = {
    # ResBlock conv2 and the Up / Down convs of a 128-channel level: two 64-channel chunks (128 x 128 x 9 fp16 = 288 KB)
    "c128": dict(args=(128, 128, 9, 128, 128, 0, False, True), chunks=[64, 64], mode="fp16", widthT=64, fprop=2, dgrad=[2], wgrad=[4]),
    # the up-path conv1 of a 128-channel level: (x, skip) concat of 128 + 128
    "cat256": dict(args=(128, 256, 9, 128, 128, 128, False, True), chunks=[64, 64, 64, 64], mode="fp16", widthT=64, fprop=4,
                   dgrad=[2, 2], wgrad=[4, 4]),
    # the last up block at a 64 / 128 boundary: chunks of 128 and 64 (128 x 64 x 9 fp16 = 144 KB fits); the dgrad packs are
    # exactly 144 KB, so they run unchunked
    "cat192": dict(args=(64, 192, 9, 128, 128, 64, False, True), chunks=[128, 64], mode="fp16", widthT=0, fprop=2, dgrad=[1, 1],
                   wgrad=[2, 1]),
    # Downsample at 128
    "down128": dict(args=(128, 128, 9, 128, 128, 0, False, True), stride=2, chunks=[64, 64], mode="fp16", widthT=64, fprop=2,
                    dgrad=[2], wgrad=[4]),
    # skip projections: split-fp16 chunks of 128 in one launch each (3 x 128 x 128 fp16 = 96 KB <= 120 KB)
    "proj256": dict(args=(128, 256, 1, 128, 128, 128, True, True), chunks=[128, 128], mode="precise", widthT=0, fprop=2,
                    dgrad=[1, 1], wgrad=[4, 4]),
    "proj192": dict(args=(64, 192, 1, 128, 128, 64, True, True), chunks=[128, 64], mode="precise", widthT=0, fprop=2, dgrad=[1, 1],
                    wgrad=[2, 1]),
    # the actor-critic's SmallResBlock conv at 128: eight one-launch split-fp16 chunks would be needed, so three passes x 2 chunks
    "ac128": dict(args=(128, 128, 9, 128, 128, 0, True, True), chunks=[64, 64], mode="three_pass", widthT=64, fprop=6, dgrad=[2],
                  wgrad=[4]),
    # the actor-critic's level changes: exactly 144 KB of weights, so unchunked, three passes
    "ac64_128": dict(args=(128, 64, 9, 64, 64, 0, True, True), chunks=[], mode="three_pass", widthT=0, fprop=3, dgrad=[1], wgrad=[2]),
    "ac128_64": dict(args=(64, 128, 9, 128, 128, 0, True, True), chunks=[], mode="three_pass", widthT=0, fprop=3, dgrad=[1], wgrad=[2]),
    # conv_in of training config D4 (60 real channels stored as 64): three passes over a padded source
    "conv_in60": dict(args=(64, 60, 9, 60, 64, 0, True, False), chunks=[], mode="three_pass", widthT=0, fprop=3, dgrad=[], wgrad=[1]),
    # conv_in into a 128-channel level 0 (15 real channels stored as 16): split-fp16 in one launch
    "conv_in15": dict(args=(128, 15, 9, 15, 16, 0, True, False), chunks=[], mode="precise", widthT=0, fprop=1, dgrad=[], wgrad=[2]),
    # conv_out over 128 channels: Cout 3 of 16, and two 64-channel blocks of activations for its weight gradient
    "conv_out": dict(args=(3, 128, 9, 128, 128, 0, False, True), chunks=[], mode="fp16", widthT=0, fprop=1, dgrad=[1], wgrad=[2]),
}
SIZES = [(5, 8, 8), (2, 24, 40), (1, 16, 16)]


def layer(name):
    return ops.ConvLayer(*LAYERS[name]["args"])


def sources(name):
    """[(stored channels, real channels, offset of its first real channel in the torch weight)] of the layer's sources."""
    cout, cin_real, taps, c0_real, c0_store, c1, split, dgrad = LAYERS[name]["args"]
    return [(c0_store, c0_real, 0)] + ([(c1, c1, c0_real)] if c1 else [])


def _covered_once(spans, total):
    cells = sorted(c for a, n in spans for c in range(a, a + n))
    assert cells == list(range(total)), (spans, total)


@pytest.mark.parametrize("name", list(LAYERS))
def test_walker_choices(name):
    e, L = LAYERS[name], layer(name)
    info = L.info
    cout, cin_real, taps, _, c0_store, c1, _, dgrad = e["args"]
    assert info["Cin"] == c0_store + c1 and info["CoutPad"] == ops.round_up(cout, 16)
    assert info["nchunks"] == len(e["chunks"])
    assert (info["precise"], info["three_pass"]) == {"fp16": (0, 0), "precise": (1, 0), "three_pass": (0, 1)}[e["mode"]]
    assert info["widthT"] == e["widthT"] and info["nsrcT"] == (len(sources(name)) if dgrad else 0)
    assert info["fprop_launches"] == e["fprop"]
    assert info["dgrad_launches"][:info["nsrcT"]] == e["dgrad"]
    assert info["wgrad_launches"][:len(sources(name))] == e["wgrad"]
    if name in ("ac64_128", "ac128_64"):   # the resident-weight limit itself: 144 KB of fp16 weights, no K split
        assert taps * info["Cin"] * info["CoutPad"] * 2 == 144 * 1024
    launches = L.fprop_plan(5, 8, 8, stride=e.get("stride", 1))
    assert [ln["C0"] for ln in launches[::3 if e["mode"] == "three_pass" else 1]] == (e["chunks"] or [c0_store])


# the statistics epilogue takes Cout in {16, 32, 64, 128}: conv_out (Cout 3) runs without
FLAGS = [(n, residual, stats) for n in LAYERS for residual, stats in [(False, False), (True, True), (False, True)]
         if not (stats and LAYERS[n]["args"][0] % 16)]


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name,residual,stats", FLAGS)
def test_forward_launches(name, size, residual, stats):
    e, L = LAYERS[name], layer(name)
    info = L.info
    cout = e["args"][0]
    b, h, w = size
    launches = L.fprop_plan(b, h, w, stride=e.get("stride", 1), residual=residual, stats=stats, out_gs=32 if stats else 0)
    assert len(launches) == e["fprop"]
    # bias and the caller's residual on the first launch only; every later launch accumulates onto out; statistics on the last
    for i, ln in enumerate(launches):
        assert ln["bias"] == (i == 0), (i, ln)
        assert ln["residual"] == (i == 0 and residual), (i, ln)
        assert ln["residual_is_out"] == (i > 0), (i, ln)
        assert ln["stats"] == (stats and i == len(launches) - 1), (i, ln)
        assert ln["Cout"] == cout and ln["CoutPad"] == info["CoutPad"]
        assert 0 <= ln["wpk"] < info["packed_bytes"] and ln["wpk"] % 256 == 0
    passes = 3 if info["three_pass"] else 1
    groups = [launches[i:i + passes] for i in range(0, len(launches), passes)]
    srcs = sources(name)
    if not info["nchunks"]:
        (first, *_), = groups
        c1 = srcs[1][0] if len(srcs) > 1 else 0
        assert (first["C0"], first["C1"]) == (srcs[0][0], c1)
        assert first["src"][:2] == [0, 1 if c1 else -1] and first["plane"][:2] == [0, 0]
    spans = {k: [] for k in range(len(srcs))}
    packs = set()
    for g in groups:
        hi = g[0]
        k = hi["src"][0]
        assert k in spans and hi["plane"][0] >= 0, hi
        spans[k].append((8 * hi["plane"][0], hi["C0"]))
        assert hi["precise"] == info["precise"]
        if info["nchunks"]:
            assert hi["C1"] == 0 and hi["src"][1] == -1
        if info["precise"]:   # the low parts of the same channels
            assert hi["src"][2:] == [2 + hi["src"][0], (3 if hi["src"][1] == 1 else -1)] and hi["plane"][2] == hi["plane"][0], hi
        else:
            assert hi["src"][2:] == [-1, -1], hi
        if passes == 3:
            # A_hi W_hi, then A_lo W_hi (the same pack, the low operand at the same plane), then A_hi W_lo (the low-part pack)
            lo_a, lo_w = g[1], g[2]
            assert lo_a["src"][0] == 2 + k and lo_a["plane"][0] == hi["plane"][0] and lo_a["wpk"] == hi["wpk"], g
            assert lo_a["C0"] == hi["C0"] and lo_a["src"][1] == (3 if hi["src"][1] == 1 else -1)
            assert lo_w["src"][:2] == hi["src"][:2] and lo_w["plane"][:2] == hi["plane"][:2] and lo_w["C0"] == hi["C0"], g
            assert lo_w["wpk"] != hi["wpk"] and not any(x["precise"] for x in g)
            packs.add(lo_w["wpk"])
        packs.add(hi["wpk"])
    assert len(packs) == len(groups) * (2 if passes == 3 else 1), "every chunk (and pass) has its own pack"
    for k, (stored, _, _) in enumerate(srcs):
        if info["nchunks"] or k == 0:
            _covered_once(spans[k] if info["nchunks"] else [(0, stored)], stored)


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", [n for n in LAYERS if LAYERS[n]["dgrad"]])
def test_dgrad_launches(name, size, accumulate):
    e, L = LAYERS[name], layer(name)
    info = L.info
    b, h, w = size
    packs = set()
    for k, (_, real, _) in enumerate(sources(name)):
        launches = L.dgrad_plan(k, b, h, w, accumulate)
        assert len(launches) == e["dgrad"][k]
        for j, ln in enumerate(launches):
            width = info["widthT"] or info["CoutPad"]
            assert ln["src"] == [0, -1, -1, -1] and ln["plane"][0] == j * width // 8, (j, ln)
            assert ln["C0"] == width and ln["C1"] == 0 and not ln["precise"]
            assert ln["Cout"] == real and ln["CoutPad"] == ops.round_up(real, 16)
            assert ln["residual_is_out"] == (accumulate or j > 0) and not ln["residual"] and not ln["bias"] and not ln["stats"]
            packs.add(ln["wpk"])
        assert sum(ln["C0"] for ln in launches) == info["CoutPad"]
    assert len(packs) == sum(e["dgrad"]), "every source and gradient chunk has its own transposed pack"


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", list(LAYERS))
def test_wgrad_blocks_tile_the_weight_once(name, size):
    e, L = LAYERS[name], layer(name)
    cout = e["args"][0]
    b, h, w = size
    for k, (stored, real, off) in enumerate(sources(name)):
        blocks = L.wgrad_plan(stored, real, off, b, h, w)
        assert len(blocks) == e["wgrad"][k]
        cells = []
        for bl in blocks:
            # gradient planes from co_off, activation planes from the block's first input channel
            assert bl["src"][:2] == [0, 1] and bl["plane"][0] == bl["co_off"] // 8 and bl["plane"][1] == (bl["ci_off"] - off) // 8, bl
            assert bl["Cg"] == min(64, ops.round_up(cout, 16) - bl["co_off"]) and bl["C0"] == min(64, stored - (bl["ci_off"] - off))
            assert bl["Cout"] <= bl["Cg"] and bl["Cin"] <= bl["C0"]
            cells += [(co, ci) for co in range(bl["co_off"], bl["co_off"] + bl["Cout"]) for ci in range(bl["ci_off"], bl["ci_off"] + bl["Cin"])]
        assert sorted(cells) == [(co, ci) for co in range(cout) for ci in range(off, off + real)], name


def test_padding_channels_are_outside_every_block():
    """Cout 3 of a 16-channel gradient operand, 15 of 16 and 60 of 64 input channels: the blocks' Cout / Cin stop at the real
    channels, so the zero (or stale) padding of an operand never reaches dW."""
    (bl,) = [x for x in layer("conv_out").wgrad_plan(64, 64, 64, 1, 8, 8)]
    assert (bl["Cg"], bl["Cout"], bl["co_off"], bl["ci_off"], bl["Cin"]) == (16, 3, 0, 64, 64)
    assert [(x["co_off"], x["Cout"], x["Cin"]) for x in layer("conv_in15").wgrad_plan(16, 15, 0, 1, 8, 8)] == [(0, 64, 15), (64, 64, 15)]
    assert [(x["C0"], x["Cin"]) for x in layer("conv_in60").wgrad_plan(64, 60, 0, 1, 8, 8)] == [(64, 60)]


def test_refusals():
    lib = _lib.lib()
    # (256 + 128) -> 128: six 64-channel chunks, more than the four an expansion holds
    with pytest.raises(RuntimeError, match="more than 4 K-split chunks"):
        ops.ConvLayer(128, 384, 9, 256, 256, 128)
    assert lib.dmd_conv_layer_create(128, 384, 9, 256, 256, 128, 0, 1) is None
    assert b"K-split chunks" in lib.dmd_last_error()
    with pytest.raises(RuntimeError, match="needs the low operand parts"):
        layer("ac128").fprop_plan(5, 8, 8, lo=False)
    with pytest.raises(RuntimeError, match="no backward-data pack"):
        layer("c128").dgrad_plan(1, 5, 8, 8)
    with pytest.raises(RuntimeError, match="no backward-data pack"):
        layer("conv_in15").dgrad_plan(0, 5, 8, 8)
    with pytest.raises(RuntimeError, match="input channels"):
        layer("cat192").wgrad_plan(128, 128, 128, 5, 8, 8)
    with pytest.raises(RuntimeError, match="more than 2 launches"):
        L = layer("ac128")
        L._PLAN_CAP = 2
        L.fprop_plan(5, 8, 8)
