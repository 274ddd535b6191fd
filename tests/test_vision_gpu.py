"""The vision half of the model (ViT over the crops, then stitch / pool / projection, then the image prefill) against an
fp64 reference at the 2B and 0.5B widths, crop by crop and row by row, and bit for bit across batches of up to 416 crops.

  * md_vision_encode, two ViT layers: the 2B (D = 1152, 16 heads, FF 4304) and the 0.5B (D = 720, 10 heads, FF 2690
    zero-padded to 2696, so every ViT GEMM ends in a partial column tile), on batches of 1, 3 and 10 crops;
  * md_vision_project on batches whose tilings cover every shape crop_tiling returns up to 12 crops, with the BOS and
    prompt rows of each image left bit-unchanged, and md_vision_project_stitched (the seam adapter's path) equal to it;
  * the full-depth 2B ViT, the projection and the image prefill at 416 crops (32 images of 12-crop tilings) and at the
    bench's 64 crops: every image's rows from one batched call equal those of the image alone, and a second launch
    repeats the first.  Every kernel on this path is batch-invariant by construction (GEMM tiles depend on N only,
    the K order is fixed per accumulator, one attention work item is one (crop, head, query tile)), so the check
    is bit equality, not a tolerance.

Reference: OracleModel.vision_encoder / vision_projection (vision.py:44-89) in fp64 on the GPU, built from the state
dict itself (the unpadded 0.5B FF, not the engine's prepared weights), rounded to bf16 wherever the reference model
rounds ("rounded") or never ("truth"); inside attention nothing is rounded.  Each crop / image must lie within REL_TOL
of the rounded reference and no further from the truth than 1.5x the rounded reference's own distance + 2e-3 (the rule
of test_decoder_gpu.py), and its worst token row within VIT_ROW_TOL / PROJ_ROW_TOL of the rounded reference.

Workspaces are filled with NaN before every call and outputs with NaN or a recorded sentinel.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

REL_TOL = 3e-2
# worst token row against the rounded reference: measured on an H100 80GB HBM3 (700 W limit) at 5.1e-3 for the ViT
# (0.5B; 4.7e-3 at 2B) and 2.0e-3 for the projection (0.5B; 1.9e-3 at 2B), bounded with a margin of 2.4x and 2.5x
VIT_ROW_TOL = 1.2e-2
PROJ_ROW_TOL = 5e-3
NAN_BYTE = 255          # 0xffff is a bf16 NaN

# every (rows, cols) tiling crop_tiling returns for up to 12 crops, with an image size that produces it
TILING_SIZES = {(1, 1): (378, 378), (2, 4): (500, 800), (4, 2): (800, 500), (3, 3): (384, 384), (2, 6): (384, 960),
                (6, 2): (960, 384), (3, 4): (671, 868), (4, 3): (883, 655), (1, 9): (406, 3637), (9, 1): (3637, 406)}


def _lib():
    from moondream_b200 import _native as N

    return N, N.lib()


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _bf(t):
    return t.to(torch.bfloat16).to(torch.float64)


def _same(t):
    return t


def _nan(shape, dtype=torch.bfloat16):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _nan_ws(eng, nbytes):
    """the engine's own workspace (one buffer for every call, so the 416-crop ViT's 7.2 GB exists once), all NaN"""
    return eng._workspace(int(nbytes)).fill_(NAN_BYTE)


def _peak():
    return f"peak allocated so far {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB"


def _bits(t):
    return t.contiguous().view(torch.int16)


def _assert_same_bits(got, want, what):
    bad = (_bits(got) != _bits(want)).reshape(got.shape[0], -1).any(dim=1)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {got.shape[0]} rows differ, first at row " \
                                f"{int(bad.nonzero()[0])}"


# ------------------------------------------------------------------------------------------------ models
def _config(name):
    """the 2B or 0.5B preset with a two-layer decoder; two ViT layers, or all 27 for "2b-27" """
    from moondream_b200 import config as C

    cfg = C.moondream_0_5b() if name == "0.5b" else C.moondream_2b()
    return C.replace(cfg, text=C.replace(cfg.text, n_layers=2),
                     vision=C.replace(cfg.vision, enc_n_layers=27 if name == "2b-27" else 2))


@pytest.fixture(scope="module")
def model(request):
    """(name, cfg, state dict, engine); the full-depth engine has KV pages for 32 image prefixes + one"""
    from moondream_b200 import synth
    from moondream_b200.engine import Engine

    name = request.param
    cfg = _config(name)
    sd = synth.synthetic_state_dict(cfg, 11)
    pages = 33 * math.ceil(cfg.text.prefix_attn / 64) if name == "2b-27" else 1
    eng = Engine(cfg, sd, max_batch=1, kv_pages=pages)
    yield name, cfg, sd, eng
    del eng, sd
    torch.cuda.empty_cache()


def _encode(eng, crops):
    """md_vision_encode into a NaN output through a NaN workspace"""
    N, lib = _lib()
    v = eng.cfg.vision
    n = crops.shape[0]
    feats = _nan((n * v.tokens_per_crop, v.enc_dim))
    ws = _nan_ws(eng, lib.md_vision_encode_workspace_bytes(eng.model, n))
    N.check(lib.md_vision_encode(eng.model, N.ptr(crops), n, N.ptr(feats), N.ptr(ws), N.current_stream()),
            "md_vision_encode")
    torch.cuda.synchronize()
    return feats


def _project(eng, feats, offsets, tilings, out, rows_per_image):
    N, lib = _lib()
    offs = torch.tensor(offsets, dtype=torch.int32, device="cuda")
    til = torch.tensor(tilings, dtype=torch.int32, device="cuda")
    ws = _nan_ws(eng, lib.md_vision_project_workspace_bytes(eng.model, len(tilings)))
    N.check(lib.md_vision_project(eng.model, N.ptr(feats), N.ptr(offs), N.ptr(til), len(tilings), N.ptr(out),
                                  rows_per_image, N.ptr(ws), N.current_stream()), "md_vision_project")
    torch.cuda.synchronize()


def _offsets(tilings):
    offs = [0]
    for th, tw in tilings:
        offs.append(offs[-1] + 1 + th * tw)
    return offs


# ------------------------------------------------------------------------------------------------ reference
class _Ref:
    """vision.py:44-89 in fp64 from the state dict, with the model's bf16 roundings or without any"""

    def __init__(self, cfg, sd, device="cuda"):
        self.v = cfg.vision
        self.sd = sd
        self.dev = device

    def w(self, key):
        return self.sd[key].to(self.dev, torch.float64)

    def _ln(self, x, prefix):
        return F.layer_norm(x, (x.shape[1],), self.w(prefix + ".weight"), self.w(prefix + ".bias"), 1e-5)

    def _lin(self, x, prefix):
        return x @ self.w(prefix + ".weight").t() + self.w(prefix + ".bias")

    def _attention(self, qkv, n):
        """scaled_dot_product_attention per crop and head, nothing rounded inside"""
        tok, H = self.v.tokens_per_crop, self.v.enc_n_heads
        D = qkv.shape[1] // 3
        hd = D // H
        out = torch.empty(qkv.shape[0], D, dtype=torch.float64, device=self.dev)
        for c in range(n):
            rows = slice(c * tok, (c + 1) * tok)
            q, k, v = (t.reshape(tok, H, hd).transpose(0, 1) for t in qkv[rows].split(D, dim=1))
            p = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(hd), dim=-1)
            out[rows] = (p @ v).transpose(0, 1).reshape(tok, D)
        return out

    def encode(self, crops_u8, rounded):
        """uint8 NHWC crops [n, S, S, 3] -> [n * 729, D]"""
        r = _bf if rounded else _same
        v = self.v
        n, P, g = crops_u8.shape[0], v.enc_patch_size, v.grid
        px = crops_u8.cpu().permute(0, 3, 1, 2)
        if rounded:      # vision.py:36-40: bf16 in place, /255, -0.5, /0.5
            px = px.to(torch.bfloat16).div_(255.0).sub_(0.5).div_(0.5).double()
        else:
            px = (px.double() / 255.0 - 0.5) / 0.5
        x = px.to(self.dev).reshape(n, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(n * g * g, 3 * P * P)
        x = r(self._lin(x, "vision.patch_emb"))
        x = r(x.view(n, g * g, -1) + self.w("vision.pos_emb")).view(n * g * g, -1)
        for i in range(v.enc_n_layers):
            p = f"vision.blocks.{i}"
            qkv = r(self._lin(r(self._ln(x, p + ".ln1")), p + ".attn.qkv"))
            a = r(self._lin(r(self._attention(qkv, n)), p + ".attn.proj"))
            x = r(x + a)
            h = r(F.gelu(r(self._lin(r(self._ln(x, p + ".ln2")), p + ".mlp.fc1")), approximate="tanh"))
            x = r(x + r(self._lin(h, p + ".mlp.fc2")))
        return r(self._ln(x, "vision.post_ln"))

    def project(self, cat, rounded):
        """the projection MLP on [global | pooled] rows (bf16) -> [rows, txt_dim]"""
        r = _bf if rounded else _same
        h = r(F.gelu(r(self._lin(cat.double(), "vision.proj_mlp.fc1")), approximate="tanh"))
        return r(self._lin(h, "vision.proj_mlp.fc2"))


def _stitch_pool(feats, offsets, tilings, cfg):
    """[global | adaptive_avg_pool2d(stitched local crops)] per image on torch CPU bf16 (the existing kernel test
    pins these bits): [n_images * 729, 2 D], plus each image's global rows and stitched map"""
    from oracle.moondream_oracle import stitch_crops

    v = cfg.vision
    g, D = v.grid, v.enc_dim
    f = feats.cpu().view(-1, g, g, D)
    cats, parts = [], []
    for i, til in enumerate(tilings):
        glob = f[offsets[i]].reshape(g * g, D)
        stitched = stitch_crops(f[offsets[i] + 1: offsets[i + 1]], til, v.overlap_margin)
        pooled = F.adaptive_avg_pool2d(stitched.permute(2, 0, 1), output_size=(g, g)).permute(1, 2, 0).reshape(g * g, D)
        cats.append(torch.cat([glob, pooled], dim=1))
        parts.append((glob, stitched))
    return torch.cat(cats).cuda(), parts


class _Worst:
    """the largest errors seen, for the summary line"""

    def __init__(self):
        self.unit = self.row = self.ratio = 0.0


def _check_units(got, rounded, truth, unit_rows, row_tol, what, worst):
    """per unit (a crop or an image) of `unit_rows` rows: REL_TOL against the rounded reference and the truth rule;
    per token row: row_tol against the rounded reference"""
    assert torch.isfinite(got.double()).all(), f"{what}: non-finite values"
    for u in range(got.shape[0] // unit_rows):
        rows = slice(u * unit_rows, (u + 1) * unit_rows)
        e_ref = rel(got[rows], rounded[rows])
        e_truth, e_own = rel(got[rows], truth[rows]), rel(rounded[rows], truth[rows])
        assert e_ref < REL_TOL, f"{what} #{u}: rel err {e_ref:.3e} against the rounded reference"
        assert e_truth <= 1.5 * e_own + 2e-3, \
            f"{what} #{u}: rel err {e_truth:.3e} against fp64 truth (rounded reference's own {e_own:.3e})"
        worst.unit = max(worst.unit, e_ref)
        worst.ratio = max(worst.ratio, e_truth / max(e_own, 1e-30))
    d = got.double() - rounded
    row_err = d.norm(dim=1) / (rounded.norm(dim=1) + 1e-30)
    r = int(row_err.argmax())
    assert row_err[r] < row_tol, f"{what}: token row {r} (#{r // unit_rows}, token {r % unit_rows}) has rel err " \
                                 f"{row_err[r]:.3e} against the rounded reference"
    worst.row = max(worst.row, row_err[r].item())


# ------------------------------------------------------------------------------------------------ (a) ViT
def _crop_kinds(eng, gen):
    """ten uint8 crops: uniform noise, all 0, all 255, noise whose lower-right part is zero (a crop that ran past the
    canvas), and six crops of a synthetic 500 x 700 image through stage_images (a global crop and five local ones)"""
    from moondream_b200 import synth

    S = eng.cfg.vision.crop_size
    noise = lambda: torch.randint(0, 256, (S, S, 3), generator=gen, dtype=torch.uint8)
    cut = noise()
    cut[250:, :] = 0
    cut[:, 300:] = 0
    own = torch.stack([noise(), torch.zeros(S, S, 3, dtype=torch.uint8), torch.full((S, S, 3), 255, dtype=torch.uint8),
                       cut]).cuda()
    staged, _, tilings = eng.stage_images([synth.synthetic_image(3, 500, 700)])
    assert staged.shape[0] >= 7, tilings
    return torch.cat([own, staged[:6]]).contiguous()


@pytest.mark.parametrize("model", ["2b", "0.5b"], indirect=True)
def test_vit_against_fp64(model):
    """md_vision_encode, two layers, batches of 10, 3 and 1 crops: each crop against the fp64 reference; a crop's rows
    have the same bits in every batch it is part of"""
    name, cfg, sd, eng = model
    gen = torch.Generator().manual_seed(2024)
    crops = _crop_kinds(eng, gen)
    ref = _Ref(cfg, sd)
    rounded, truth = ref.encode(crops, True), ref.encode(crops, False)
    tok = cfg.vision.tokens_per_crop
    worst = _Worst()
    full = _encode(eng, crops)
    _check_units(full, rounded, truth, tok, VIT_ROW_TOL, f"ViT {name} batch 10", worst)
    for lo, hi in ((3, 6), (9, 10)):
        part = _encode(eng, crops[lo:hi].contiguous())
        _check_units(part, rounded[lo * tok: hi * tok], truth[lo * tok: hi * tok], tok, VIT_ROW_TOL,
                     f"ViT {name} crops {lo}..{hi - 1}", worst)
        _assert_same_bits(part, full[lo * tok: hi * tok], f"ViT {name}: crops {lo}..{hi - 1} alone vs in the batch of 10")
    print(f"ViT {name}: worst per-crop rel err {worst.unit:.2e}, worst row {worst.row:.2e}, "
          f"worst ratio to the rounded reference's distance from truth {worst.ratio:.3f}; {_peak()}")


# ------------------------------------------------------------------------------------------------ (b) projection
@pytest.mark.parametrize("prompt_rows", [0, 7], ids=["rows730", "rows737"])
@pytest.mark.parametrize("model", ["2b", "0.5b"], indirect=True)
def test_projection_against_fp64(model, prompt_rows):
    """md_vision_project on ten images, one of every tiling, from random bf16 features: the 729 rows of each image
    against the fp64 projection of the reference's stitch + pool; the BOS row and the prompt rows keep their sentinel
    bits; md_vision_project_stitched of each image gives that image's rows bit for bit"""
    from moondream_b200.image_crops import crop_tiling

    N, lib = _lib()
    name, cfg, sd, eng = model
    v, t = cfg.vision, cfg.text
    for til, size in TILING_SIZES.items():
        assert crop_tiling(size, v.overlap_margin, v.max_crops) == til, (size, til)
    tilings = list(TILING_SIZES)
    offsets = _offsets(tilings)
    tok, D, n_img = v.tokens_per_crop, v.enc_dim, len(tilings)
    gcu = torch.Generator(device="cuda").manual_seed(7 + prompt_rows + D)
    feats = torch.randn(offsets[-1] * tok, D, generator=gcu, device="cuda").bfloat16()
    rows = t.prefix_attn + prompt_rows
    sentinel = torch.randn(n_img * rows, t.dim, generator=gcu, device="cuda").bfloat16()
    out = sentinel.clone()
    _project(eng, feats, offsets, tilings, out, rows)

    img = torch.zeros(n_img, rows, dtype=torch.bool, device="cuda")
    img[:, 1: t.prefix_attn] = True
    img = img.view(-1)
    _assert_same_bits(out[~img], sentinel[~img], f"projection {name}: BOS / prompt rows")
    got = out[img]
    cat, parts = _stitch_pool(feats, offsets, tilings, cfg)
    ref = _Ref(cfg, sd)
    worst = _Worst()
    _check_units(got, ref.project(cat, True), ref.project(cat, False), tok, PROJ_ROW_TOL, f"projection {name} rows {rows}",
                 worst)

    for i, (glob, stitched) in enumerate(parts):
        one = _nan((tok, t.dim))
        ws = _nan_ws(eng, lib.md_vision_project_workspace_bytes(eng.model, 1))
        g0, st = glob.cuda().contiguous(), stitched.cuda().contiguous()
        N.check(lib.md_vision_project_stitched(eng.model, N.ptr(g0), N.ptr(st), st.shape[0],
                                               st.shape[1], N.ptr(one), N.ptr(ws), N.current_stream()),
                "md_vision_project_stitched")
        torch.cuda.synchronize()
        _assert_same_bits(one, got[i * tok: (i + 1) * tok], f"projection {name}: stitched path of tiling {tilings[i]}")
    print(f"projection {name} rows {rows}: worst per-image rel err {worst.unit:.2e}, worst row {worst.row:.2e}, "
          f"worst ratio to the rounded reference's distance from truth {worst.ratio:.3f}; {_peak()}")


# ------------------------------------------------------------------------------------------------ (c) batch invariance
def _batch(eng, kind):
    """(crops, offsets, tilings): 32 images of 12-crop tilings (416 crops), or the bench's 32 images at 378 x 378"""
    from moondream_b200 import synth

    if kind == "bench":
        return eng.stage_images([synth.synthetic_image(i, 378, 378) for i in range(32)])
    tilings = [((3, 4), (4, 3), (2, 6), (6, 2))[i % 4] for i in range(32)]
    offsets = _offsets(tilings)
    S = eng.cfg.vision.crop_size
    gen = torch.Generator().manual_seed(416)
    crops = torch.randint(0, 256, (offsets[-1], S, S, 3), generator=gen, dtype=torch.uint8).cuda()
    return crops, offsets, tilings


@pytest.mark.parametrize("kind", ["crops416", "bench"])
@pytest.mark.parametrize("model", ["2b-27"], indirect=True)
def test_batch_invariance(model, kind):
    """full-depth 2B ViT, projection and image prefill: each image's feature rows, embeddings, hidden rows and prefix
    K/V from one batched call equal, bit for bit, those of the image alone; a second launch repeats the first"""
    N, lib = _lib()
    name, cfg, sd, eng = model
    t, v = cfg.text, cfg.vision
    tok = v.tokens_per_crop
    crops, offsets, tilings = _batch(eng, kind)
    n_img = len(tilings)
    assert n_img == 32 and offsets[-1] == (416 if kind == "crops416" else 64)

    feats = _encode(eng, crops)
    assert bool(torch.isfinite(feats).all()), "non-finite ViT features"
    sentinel = torch.randn(n_img * t.prefix_attn, t.dim, device="cuda").bfloat16()
    emb = sentinel.clone()
    _project(eng, feats, offsets, tilings, emb, 0)
    emb2 = sentinel.clone()
    _project(eng, feats, offsets, tilings, emb2, 0)
    _assert_same_bits(emb2, emb, f"{kind}: second projection launch")
    del emb2
    emb = emb.view(n_img, t.prefix_attn, t.dim)[:, 1:]
    assert bool(torch.isfinite(emb).all()), "non-finite projected rows"

    def encode(c, offs, tils):
        _nan_ws(eng, lib.md_vision_encode_workspace_bytes(eng.model, offs[-1]))
        out = eng.encode_crops(c, offs, tils, return_hidden=True)
        torch.cuda.synchronize()
        return out

    held = []          # the KV pages go back even when a check fails, so the next batch still finds them
    try:
        # encode_crops launches md_vision_encode and md_vision_project again on the same batch: the determinism check
        prefixes, feats_b, emb_b, hidden_b = encode(crops, offsets, tilings)
        held += prefixes
        _assert_same_bits(feats_b, feats, f"{kind}: second ViT launch (inside encode_crops)")
        del feats_b
        _assert_same_bits(emb_b.reshape(-1, t.dim), emb.reshape(-1, t.dim), f"{kind}: embeddings inside encode_crops")
        hidden_b = hidden_b.view(n_img, t.prefix_attn, t.dim)
        for i in range(n_img):
            lo, hi = offsets[i], offsets[i + 1]
            p1, f1, e1, h1 = encode(crops[lo:hi].contiguous(), [0, hi - lo], [tilings[i]])
            held += p1
            what = f"{kind}: image {i} (tiling {tilings[i]}) alone vs in the batch"
            _assert_same_bits(f1, feats[lo * tok: hi * tok], f"{what}, ViT features")
            _assert_same_bits(e1[0], emb[i], f"{what}, projected embeddings")
            _assert_same_bits(h1, hidden_b[i], f"{what}, prefill hidden rows")
            alone, batched = eng.prefix_kv_tensors(p1[0]), eng.prefix_kv_tensors(prefixes[i])
            for layer, ((k1, v1), (kb, vb)) in enumerate(zip(alone, batched)):
                _assert_same_bits(k1[0].transpose(0, 1), kb[0].transpose(0, 1), f"{what}, layer {layer} K")
                _assert_same_bits(v1[0].transpose(0, 1), vb[0].transpose(0, 1), f"{what}, layer {layer} V")
            p1[0].release()
    finally:
        for p in held:
            p.release()
    print(f"batch invariance {kind}: {n_img} images, {offsets[-1]} crops; {_peak()}")
