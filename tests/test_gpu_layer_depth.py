"""The persistent tile loops of the conv GEMM (gemm_tc.cu) and the fused residual pair (pair_tc.cu) at production depth,
against the float64 references of oracle/layers.py.

Both kernels run grid = min(tiles, SMs) CTAs, and each CTA loops over tile = blockIdx.x + j * gridDim.x.  State carries from
one tile of a CTA to the next: the operand ring's slot and phase, the residual TMA run-ahead into the next tiles (empty
varlen tiles included), the per-column-block epilogue constants, a pending TMA store; in the pair the five-slot A-tap ring,
the correction-tile stages and the conv_a issued ahead for the next tile that is not empty.  test_gpu_layers.py checks every
configuration at one to three tiles per CTA; the cases here run at least DEPTH tiles on every CTA (sized from the SM
count), change column block inside a CTA, and run varlen sets whose CTAs meet live -> empty -> ... -> live tile sequences.
Every element is held to the same bound as in test_gpu_layers.py: depth changes no element's arithmetic."""
import resource
import time

import pytest
import torch

import test_gpu_layers as G
from oracle import layers as R
from test_gpu_layers import BY_NAME, CONV2D, CONVT1D, CONVT2D, PAIR, TOL, C, eng, run_and_check  # noqa: F401 (eng: fixture)

pytestmark = pytest.mark.gpu

DEPTH = 16                    # tiles per CTA every deep case reaches at least
GEMM_BM, PAIR_ROWS = 128, 126   # GEMM tile rows (gemm.cuh); valid output rows of a pair tile (pair_tc.cu)

REPORTS = {}                  # case name -> (case, reported launch configuration)


class RefClock:
    """Wall and CPU time spent in the float64 references (outermost calls of the wrapped functions only)."""

    def __init__(self):
        self.depth, self.wall, self.cpu = 0, 0.0, 0.0

    def wrap(self, f):
        def timed(*a, **kw):
            if self.depth:
                return f(*a, **kw)
            self.depth += 1
            t, p = time.perf_counter(), time.process_time()
            try:
                return f(*a, **kw)
            finally:
                self.wall += time.perf_counter() - t
                self.cpu += time.process_time() - p
                self.depth -= 1
        return timed


REF = RefClock()


@pytest.fixture(scope="module", autouse=True)
def timed_references():
    """Every float64 reference run_and_check evaluates (test_gpu_layers.reference, and oracle.layers' pair / conv1d that
    check_pair calls) adds its time to REF."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(G, "reference", REF.wrap(G.reference))
        mp.setattr(R, "pair", REF.wrap(R.pair))
        mp.setattr(R, "conv1d", REF.wrap(R.conv1d))
        yield


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------ tile geometry, as plan.cu's Builder::gemm / pair_setup
def gemm_geometry(c):
    """(rows_in, N, bn) of a GEMM case: the GEMM rows per image, the packed weight's columns and the column tile."""
    kind, terms, cout = c["kind"], c.get("terms", 1), c["cout"]
    if kind in (CONV2D, CONVT2D):
        rows, N = c["H"] * (c["W"] + 1), cout if kind == CONV2D else 4 * cout
    elif kind == CONVT1D:
        rows, N = c["L"] + 1, c["stride"] * cout
    else:
        rows, N = c["L"], cout
    bn = 128 if terms == 1 and N % 128 == 0 else 64 if N % 64 == 0 else 32
    return rows, N, bn


def tile_layout(c):
    """(tiles per image, column tiles, a function tile -> live) of case c: a tile is empty when its first row lies at or past
    its image's row_valid (tile_is_empty in gemm.cuh, tile_at in pair_tc.cu)."""
    rv = c.get("row_valid")
    s, pad = 1, 0
    if c["kind"] == PAIR:
        per, n_col, rows_per = -(-c["L"] // PAIR_ROWS), 1, PAIR_ROWS
    else:
        rows, N, bn = gemm_geometry(c)
        n_col, rows_per = N // bn, GEMM_BM
        per = -(-rows // GEMM_BM) * n_col
        if c["kind"] == CONVT1D:      # row_valid counts output rows: the tile's first one is stride * m0 - pad
            s, pad = c["stride"], c["stride"] // 2 + c["stride"] % 2

    def live(tile):
        img, t = divmod(tile, per)
        return rv is None or (t // n_col) * rows_per * s - pad < rv[img]
    return per, n_col, live


def changes_column(c, tiles, grid):
    """A CTA's consecutive tiles lie `grid` apart, so they move to another column block (the epilogue reloads its per-column
    constants) when the CTA runs more than one tile and the column tiles do not divide the grid."""
    return tiles > grid and grid % tile_layout(c)[1] != 0


def has_live_empty_live(c, grid):
    """Some CTA runs a live tile, then one or more empty tiles, then a live tile again."""
    per, _, live = tile_layout(c)
    total = c.get("n_img", 1) * per
    for b in range(grid):
        seq = [live(t) for t in range(b, total, grid)]
        s = "".join("L" if x else "e" for x in seq)
        if "Le" in s and "L" in s[s.index("Le") + 1:]:
            return True
    return False


def deep(name, base, rv=None, hv=None, depth=DEPTH, **kw):
    """(name, make): make(sms) is case `base` of test_gpu_layers.py (with kw) on as many images as give every CTA at least
    `depth` tiles; rv / hv: a row_valid / head_valid pattern repeated over the images (a varlen set)."""
    def make(sms):
        c = dict(BY_NAME[base], **kw)
        c["name"] = name
        per = tile_layout(dict(c, row_valid=None))[0]
        n = -(-depth * sms // per)
        if rv is not None:
            n = -(-n // len(rv)) * len(rv)
        c["n_img"] = n
        c["row_valid"] = None if rv is None else list(rv) * (n // len(rv))
        if hv is not None:
            n = -(-n // len(hv)) * len(hv)
            c["n_img"], c["head_valid"] = n, list(hv) * (n // len(hv))
        return c
    return name, make


def pair(name, tiles, n_img=1, rv=None, **kw):
    """(name, make): a C = 64 fused pair of n_img images of L rows, L sized from the SM count: tiles(sms) -> (tiles per
    image, valid rows of the last tile), rv(L) -> row_valid."""
    def make(sms):
        per, last_rows = tiles(sms)
        L = (per - 1) * PAIR_ROWS + last_rows
        return C(name, PAIR, n_img=n_img, L=L, row_valid=None if rv is None else rv(L), **kw)
    return name, make


# ------------------------------------------------------------------ the deep cases
# Each entry: (name, make(sms), claims).  claims: "varlen" = some CTA runs live -> empty -> ... -> live.  Whether a case's
# CTAs change column block follows from its column tiles and the SM count (changes_column); the coverage test below asks
# for it wherever a plan launch does it.
VARLEN4 = lambda L: [L, L // 3 + 1, 1, L - 1]      # noqa: E731  a full image, a third, one row, all but one row
DEEP = [
    # ---- fused pair, one image: every CTA runs DEPTH tiles (one CTA one more), at the dilations of the three stacks
    (*pair("pair.deep_d1", lambda s: (DEPTH * s + 1, 100), dilation=1), ()),
    (*pair("pair.deep_d27", lambda s: (DEPTH * s + 1, 100), dilation=27), ()),
    (*pair("pair.deep_d243", lambda s: (DEPTH * s + 1, 100), dilation=243), ()),
    (*pair("pair.deep_last", lambda s: (DEPTH * s + 1, 100), dilation=243, last=True, out_row0=3, out_slack=6), ()),
    # ---- the tail of the loop: one CTA runs one more tile than the others / all but one CTA do
    (*pair("pair.tail_plus1", lambda s: (DEPTH * s + 1, 63), dilation=9), ()),
    (*pair("pair.tail_minus1", lambda s: ((DEPTH + 1) * s - 1, PAIR_ROWS), dilation=3), ()),
    # ---- varlen: four images of L rows, rows [L, L / 3 + 1, 1, L - 1]; empty runs, a one-row image, live after empty
    (*pair("pair.varlen_deep", lambda s: (4 * s + 5, 109), n_img=4, rv=VARLEN4, dilation=9), ("varlen",)),
    (*pair("pair.varlen_deep_last", lambda s: (4 * s + 5, 109), n_img=4, rv=VARLEN4, dilation=243, last=True, out_row0=3,
           out_slack=6), ("varlen",)),
    # ---- GEMM column-block changes: the condition net (4 / 8 column tiles at 1 / 3 terms), the stem, the up-samplers
    (*deep("cond.deep_t1", "cond.tv42_t1", L=1006), ()),
    (*deep("cond.deep_t3", "cond.tv42_t3", L=1006), ()),
    (*deep("cond.deep_t1_varlen", "cond.varlen_t1", rv=[1006, 336, 1, 1005], L=1006), ("varlen",)),
    (*deep("cond.deep_t3_varlen", "cond.varlen_t3", rv=[1006, 336, 1, 1005], L=1006), ("varlen",)),
    (*deep("stem.deep_k7", "stem.k7", L=1006), ()),
    (*deep("stem.deep_k7_t3", "stem.k7_t3", L=1006), ()),
    (*deep("up.deep_s7_ar", "up.s7_ar_tma", L=1006), ()),
    (*deep("up.deep_s7_ar_2", "up.s7_ar_tma_2img"), ()),
    (*deep("up.deep_s7_ar_varlen", "up.s7_ar_tma_varlen", rv=[2058, 687, 1, 2057], L=294), ("varlen",)),
    (*deep("up.deep_s3_ar", "up.s3_ar_tma_c64"), ()),
    (*deep("up.deep_s3_ar_varlen", "up.s3_ar_varlen", rv=[600, 201, 1, 597]), ("varlen",)),
    (*deep("up.deep_s3_t3", "up.s3_t3"), ()),
    (*deep("up.deep_s3_t3_varlen", "up.s3_t3_varlen", rv=[900, 301, 1, 899]), ("varlen",)),
    # ---- the vocoder's 1-term res.a signature (the stem's) and its 3-term stem / res.a, varlen
    (*deep("stem.deep_k7_varlen", "stem.k7", rv=[1006, 336, 1, 1005], L=1006), ("varlen",)),
    (*deep("stem.deep_k7_t3_varlen", "stem.k7_t3", rv=[1006, 336, 1, 1005], L=1006), ("varlen",)),
    # ---- the 3-term up-samplers at stride 7 (s * cout / 64 column tiles)
    (*deep("up.deep_s7_t3", "up.s3_t3", stride=7, cin=256, cout=128), ()),
    (*deep("up.deep_s7_t3_varlen", "up.s3_t3_varlen", rv=[2100, 701, 1, 2099], stride=7, cin=256, cout=128), ("varlen",)),
    # ---- residual run-ahead at depth: planes by TMA, the (a, r) stream of the C >= 128 stacks, the UNet's fp32 stream
    (*deep("res_b.deep_planes_c128", "res_b.planes_c128"), ()),
    (*deep("res_b.deep_planes_c128_varlen", "res_b.planes_c128", rv=[1000, 334, 1, 999]), ("varlen",)),
    (*deep("res_b.deep_planes_c64_t3", "res_b.planes_c64_t3"), ()),
    (*deep("res_b.deep_planes_c64_t3_varlen", "res_b.planes_c64_t3_varlen", rv=[500, 167, 1, 499]), ("varlen",)),
    (*deep("res_b.deep_ar_c128", "res_b.ar_c512", L=1000, cin=128, cout=128), ()),
    (*deep("res_b.deep_ar_c128_varlen", "res_b.ar_c128_varlen", rv=[700, 234, 1, 699]), ("varlen",)),
    (*deep("res_b.deep_ar_c256", "res_b.ar_c256", L=1000), ()),
    (*deep("res_b.deep_ar_c256_varlen", "res_b.ar_c256", rv=[1000, 334, 1, 999], L=1000), ("varlen",)),
    (*deep("res_b.deep_planes_last_c128_t3", "res_b.planes_last_c128_t3"), ()),
    (*deep("res_b.deep_planes_last_c128_t3_varlen", "res_b.planes_last_c128_t3_varlen", rv=[500, 167, 1, 499]), ("varlen",)),
    (*deep("res_b.deep_planes_c512_t3", "res_b.planes_c512_t3"), ()),
    (*deep("res_b.deep_planes_c512_t3_varlen", "res_b.planes_c512_t3", rv=[300, 101, 1, 299]), ("varlen",)),
    (*deep("res_b.deep_planes_last_c512_t3", "res_b.planes_last_c256_t3", cin=512, cout=512), ()),
    (*deep("res_b.deep_planes_last_c512_t3_varlen", "res_b.planes_last_c256_t3_varlen", rv=[300, 101, 1, 299], cin=512,
           cout=512), ("varlen",)),
    (*deep("res_b.deep_last_of_stack", "res_b.last_of_stack"), ()),
    (*deep("res_b.deep_last_of_stack_varlen", "res_b.last_of_stack_varlen", rv=[500, 167, 1, 499]), ("varlen",)),
    (*deep("conv2_res.deep_c32", "conv2_res.c32_varlen", rv=None, H=8, W=127), ()),
    (*deep("conv2_res.deep_c32_varlen", "conv2_res.c32_varlen", rv=[1024, 342, 1, 1023], H=8, W=127), ("varlen",)),
    # ---- the mel UNet's conv GEMMs at the 32- and 64-channel levels (the levels whose CTAs run many tiles), uniform and
    #      varlen: varlen rows are whole time frames of W + 1 = 128 or 64 rows
    (*deep("conv1.deep_c32", "conv1.mel_l0", H=8), ()),
    (*deep("conv1.deep_c32_varlen", "conv1.mel_l0_varlen", rv=[1024, 384, 128, 896]), ("varlen",)),
    (*deep("conv1.deep_c64", "conv1.varlen", rv=None), ()),
    (*deep("conv1.deep_c64_varlen", "conv1.varlen", rv=[512, 192, 64, 448]), ("varlen",)),
    (*deep("conv1.deep_dec6_b2", "conv1.dec6_b2", H=8), ()),
    (*deep("conv1.deep_dec6_b2_varlen", "conv1.dec6_b2_varlen", rv=[1024, 384, 128, 896], H=8), ("varlen",)),
    (*deep("conv1.deep_enc2_b1", "conv1.enc2_b1", H=8), ()),
    (*deep("conv1.deep_enc2_b1_varlen", "conv1.enc2_b1_varlen", rv=[512, 192, 64, 448], H=8), ("varlen",)),
    (*deep("conv2_sc.deep_enc2_b1", "conv2_sc.enc2_b1", H=8), ()),
    (*deep("conv2_sc.deep_enc2_b1_varlen", "conv2_sc.enc2_b1_varlen", rv=[512, 192, 64, 448], H=8), ("varlen",)),
    (*deep("conv2_sc.deep_dec6_b2", "conv2_sc.dec6_b2", H=8), ()),
    (*deep("conv2_sc.deep_dec6_b2_varlen", "conv2_sc.dec6_b2_varlen", rv=[1024, 384, 128, 896], H=8), ("varlen",)),
    (*deep("conv2_res.deep_c64", "conv2_res.varlen_empty_tiles", rv=None, H=8), ()),
    (*deep("conv2_res.deep_c64_varlen", "conv2_res.varlen_empty_tiles", rv=[512, 192, 64, 448], H=8), ("varlen",)),
    (*deep("conv2_res.deep_dec_b5_relu", "conv2_res.dec_b5_relu", H=8), ()),
    (*deep("conv2_res.deep_dec_b5_relu_varlen", "conv2_res.dec_b5_relu_varlen", rv=[512, 192, 64, 448], H=8), ("varlen",)),
    (*deep("skip_concat.deep_enc1_b4", "skip_concat.enc1_b4", H=8), ()),
    (*deep("skip_concat.deep_enc1_b4_varlen", "skip_concat.enc1_b4_varlen", rv=[1024, 384, 128, 896], H=8), ("varlen",)),
    (*deep("skip_concat.deep_enc_b4", "skip_concat.enc_b4", H=8), ()),
    (*deep("skip_concat.deep_enc_b4_varlen", "skip_concat.enc_b4_varlen", rv=[512, 192, 64, 448], H=8), ("varlen",)),
    (*deep("head.deep_mel", "head.mel", hv=[7, 7]), ()),
    (*deep("head.deep_mel_varlen", "head.mel_varlen", rv=[1024, 384, 128, 896], hv=[7, 3, 1, 7]), ("varlen",)),
    # ---- the other maps at depth: ConvTranspose2d (row-major stores into the concat buffer; the decoder's up-sampling
    #      into 128 channels has 4 * 128 / 64 column tiles, and its BN scale / shift index wraps as co mod cout) and a GRU
    #      input projection
    (*deep("convt2d.deep_dec4", "convt2d.mel_time_only", cin=256, cout=128), ()),
    (*deep("convt2d.deep_dec4_varlen", "convt2d.time_only_varlen", rv=[256, 96, 32, 224], H=8, W=31, cin=256, cout=128),
     ("varlen",)),
    (*deep("convt2d.deep_both", "convt2d.v2_both", H=2, W=127), ()),
    (*deep("convt2d.deep_time_only", "convt2d.mel_time_only"), ()),
    (*deep("convt2d.deep_both_varlen", "convt2d.time_only_varlen", rv=[512, 192, 64, 448], H=8, W=63, both=1, out_slack=0),
     ("varlen",)),
    (*deep("bigru.deep_gru0.ih_T6001", "bigru.gru0.ih", L=6001), ()),
]
DEEP_BY_NAME = {n: (make, claims) for n, make, claims in DEEP}


@pytest.fixture(scope="module")
def sms():
    return sm_count()


def run_deep(eng, name, sms):
    make, claims = DEEP_BY_NAME[name]
    c = make(sms)
    t0, p0 = time.perf_counter(), time.process_time()
    worst, rep = run_and_check(eng, c)
    wall, cpu = time.perf_counter() - t0, time.process_time() - p0
    REPORTS[name] = (c, rep)
    return c, rep, worst, claims, wall, cpu


@pytest.mark.parametrize("name", [n for n, _, _ in DEEP])
def test_deep_layer_matches_float64(eng, sms, name):
    c, rep, worst, claims, wall, cpu = run_deep(eng, name, sms)
    tiles, grid = rep["tiles"], rep["grid"]
    per, n_col, _ = tile_layout(c)
    print(f"{name}: tiles {tiles} / grid {grid} = {tiles / grid:.2f} per CTA, bn {rep['bn']}, {n_col} column tiles "
          f"({'changes' if changes_column(c, tiles, grid) else 'keeps'} column block), n_img {c.get('n_img', 1)}; "
          f"max err / bound = {worst:.3e} (tol {TOL[rep['terms']]:.1e}); case {wall:.1f} s wall, {cpu:.1f} s CPU; "
          f"references so far {REF.wall:.1f} s wall, {REF.cpu:.1f} s CPU  sig {rep['sig']}")
    # the launch is the one the case was sized for, and every CTA runs at least DEPTH tiles
    assert tiles == c.get("n_img", 1) * per, (tiles, per)
    assert grid == min(tiles, sms)
    assert tiles // grid >= DEPTH, (tiles, grid)
    if c["kind"] != PAIR:
        assert rep["bn"] == gemm_geometry(c)[2]
    if "varlen" in claims:
        assert has_live_empty_live(c, grid)


# ------------------------------------------------------------------ depth coverage of the plans' launches
DEPTH_PLAN_BATCH, DEPTH_PLAN_FRAMES = 32, 1001       # 32 clips of 10 s (BASELINE config 2)


def deep_plan_sweep():
    """[(plan, label, signature, tiles, grid, col_tiles)] of every GEMM / fused-pair launch of the GSR plan (mel UNet + vocoder
    at 1 and 3 terms), uniform and varlen, at 32 clips x 1001 frames.  Plans are built, not run, one at a time, each freed
    before the next.  The GSR plan's device buffers at that shape with the 3-term vocoder (the larger of the two builds)
    must leave a quarter of the device free."""
    from test_gpu_layers import PLAN_NAMES
    from voicefixer_main_b200.model import Engine
    from voicefixer_main_b200.weights import make_state
    e = Engine("cuda:0")
    out = []
    try:
        e.load_state(make_state(1234), need=("unet", "vocoder"))
        for terms in (1, 3):
            e.set_option("vocoder_terms", terms)
            for kind in (0, 2):
                recs = e.selftest_plan_gemms(kind, DEPTH_PLAN_BATCH, DEPTH_PLAN_FRAMES, tile_loop=True)
                out += [(f"{PLAN_NAMES[kind]}.voc{terms}", *r) for r in recs]
        ws = e.workspace_bytes(DEPTH_PLAN_BATCH, (DEPTH_PLAN_FRAMES - 1) * 441)
        total = torch.cuda.get_device_properties(0).total_memory
        rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20
        print(f"GSR plan at {DEPTH_PLAN_BATCH} x {DEPTH_PLAN_FRAMES} frames: {ws / 2**30:.1f} GiB of device buffers and "
              f"weights ({total / 2**30:.0f} GiB on the device); host peak RSS {rss:.1f} GiB")
        assert ws < total * 3 // 4
        e.check_errors()
    finally:
        e.close()
    return out


def test_deep_cases_cover_every_deep_launch(eng, sms):
    """Every GEMM / fused-pair launch of the GSR plans at 32 x 10 s whose CTAs run more than one tile is covered by a deep
    case above with its configuration signature that runs at least min(DEPTH, the launch's tiles per CTA) tiles per CTA;
    where the launch's CTAs change column block the case's do too, and where the launch is varlen (so is its signature) some
    CTA of the case runs live -> empty -> ... -> live.  The pair cases reach the loop shapes a signature does not name: the
    three stacks' dilations 1, 27 and 243 at depth, and totals of k * grid + 1 and k * grid - 1 tiles.  So the steady state
    of each configuration the product runs deep is checked against float64."""
    for name, _, _ in DEEP:
        if name not in REPORTS:
            run_deep(eng, name, sms)
    print(f"float64 references of the {len(DEEP)} deep cases: {REF.wall:.1f} s wall, {REF.cpu:.1f} s CPU")
    sweep = deep_plan_sweep()
    deep_launches = [s for s in sweep if s[3] > s[4]]
    assert len(sweep) > 100 and deep_launches and all(s[2] for s in sweep)
    cover = {}
    for name, (c, rep) in REPORTS.items():
        t, g = rep["tiles"], rep["grid"]
        cover.setdefault(rep["sig"], []).append((t / g, changes_column(c, t, g), has_live_empty_live(c, g), name))
    uncovered, sole = [], {}
    for plan, label, sig, tiles, grid, col_tiles in deep_launches:
        need = min(DEPTH, tiles / grid)
        col = grid % col_tiles != 0
        varlen = sig.endswith("varlen=1")
        ok = [name for depth, c_col, c_run, name in cover.get(sig, [])
              if depth >= need and (c_col or not col) and (c_run or not varlen)]
        print(f"{plan}:{label}: {tiles} tiles / grid {grid} = {tiles / grid:.2f}, {col_tiles} column tiles"
              f"{' (changes column block)' if col else ''}  -> {', '.join(ok) or 'NONE'}  ({sig})")
        if not ok:
            uncovered.append(f"{plan}:{label} ({tiles / grid:.2f} tiles per CTA, {col_tiles} column tiles on a grid of {grid})"
                             f"\n    {sig}")
        elif len(ok) == 1:
            sole.setdefault(ok[0], []).append(f"{plan}:{label}")
    for name, labels in sorted(sole.items()):
        print(f"{name}: the only deep case of {len(labels)} launches")
    assert not uncovered, "deep plan launches whose configuration no deep case runs at their depth:\n" + "\n".join(uncovered)
    pairs = [(c, rep["tiles"], rep["grid"]) for c, rep in REPORTS.values() if c["kind"] == PAIR]
    dils = {c["dilation"] for c, t, g in pairs if c.get("row_valid") is None and not c.get("last") and t // g >= DEPTH}
    assert {1, 27, 243} <= dils, dils
    for rem in (1, -1):         # one CTA runs one tile more than the rest / one CTA runs one tile fewer
        assert any((t - rem) % g == 0 and t // g >= 10 for c, t, g in pairs), rem
