"""The benchmarked plan -- YOLOX-s, 64 images of 640 x 640 -- call by call, on the geometries its own training step and inference pass use.

At this size the host planning of the convolution GEMMs takes branches that small replays never reach: the persistent forward / data-
gradient kernels give each CTA dozens of 128-pixel tiles (their loads wrap around the TMA ring many times and their BatchNorm statistics
add up in shared memory over the whole walk), and the weight gradient's split-K is limited by occupancy, with a ragged last split.  The
module records one train_step() and one eval_forward() of YoloxEngine(64, 640, 640) through a stand-in library handle, mirrors the host
arithmetic of csrc/conv_api.cu for every recorded GEMM (printed by test_recording_is_complete with -s) and then checks:

  * every distinct GEMM geometry, replayed on fresh buffers against fp64 with the bound of tests/test_convnext_plan_gpu.py (its fp64
    references run in batch chunks, so a case needs a few GB of device memory beyond its operands);
  * exact-integer probes of the pixel-long sums: the weight gradients (plain and pixel-grouped, accumulate 0 and 1) and the BatchNorm
    statistics of every training forward, on {0, 1} operands.  Every partial sum is then a non-negative integer below 2^20, exact in
    fp32, in the fp64 atomics and in the split reduction, so the kernel must equal the fp64 reference bit for bit, and one dropped or
    repeated pixel block, tap, split or tile is off by at least 1.  At K = 6.5 M pixels the random-operand bound cannot see such a
    defect (tests/test_headline_plan_tol_cpu.py shows both sides);
  * every BatchNorm of a real 64 x 640 x 640 step on the operands the engine gave it (tests/test_train_bn_gpu.py's per-layer checks, the
    statistics bound taken from the mirrored per-CTA tile walk), the prediction-bias gradients, SimOTA and the losses against the oracle,
    the Focus preprocessing, the head decode, and the eval-path BatchNorm;
  * SPP forward and backward at the plan's 64 x 20 x 20 x 256.
"""
import ctypes
import math

import pytest
import torch

from test_convnext_plan_gpu import (RUN, SENTINEL, WORST, _act, _case_of, _fold_mask, _g, _guard_ok, _guarded, _lib, _out_view,
                                    _outside_same, _sl, _yolox_names, conv_ref, wgrad_ref)
from test_engine_headline_gpu import _check_assign_and_losses
from test_fixed_order_gpu import check_spp_pool
from test_train_bn_gpu import (U32, _check_apply, _choose_tile, _fail, _heads, build_step, check_every_batchnorm, _check_head_bias)

from oracle import yolox_oracle as orc

pytestmark = pytest.mark.gpu

BATCH, SIZE = 64, 640
EXACT_LIMIT = 2 ** 20
PEAK = {}  # case kind -> most device memory one case allocated beyond what was live before it (printed at the end with -s)


# ------------------------------------------------------------------------------------------------------------------------------------
# host planning of csrc/conv_api.cu, restated
# ------------------------------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_block_k(c):
    return 64 if c % 64 == 0 else (32 if c % 32 == 0 else (16 if c % 16 == 0 else 0))


def pick_block_n(c):
    return 128 if c > 64 else (64 if c > 32 else (32 if c > 16 else 16))


def conv_min_ctas(bn, bk):
    return 1 if (bn >= 128 or bk == 16) else 2


def gemm_plan(case, sms):
    """persistent forward / data-gradient launch (launch_conv_inst): work items (pixel tiles x output-parity phases), column tiles,
    groups of CTAs per column tile, and the most work items one CTA walks"""
    fn = case["fn"]
    if fn == "dgrad":
        n, h, w, cin = case["gdz"][:4]
        cout, phases = case["gdx"][3], 4 if case["s"] == 2 else 1
    elif fn == "pred":
        n, h, w, cin = case["gx"][:4]
        cout, phases = case["cout"], 1
    else:
        out = case["gz"] if fn == "fwd" else case["go"]
        n, h, w = out[:3]
        cin, cout, phases = case["gx"][3], out[3], 1
    bk, bn = pick_block_k(cin), pick_block_n(cout)
    m_tiles = _choose_tile(n, h, w) * phases
    n_tiles = -(-cout // bn)
    groups = min(max(1, conv_min_ctas(bn, bk) * sms // n_tiles), m_tiles)
    if phases == 4 and groups > 1 and groups % 2 == 0:
        groups -= 1
    return dict(bn=bn, bk=bk, phases=phases, m_tiles=m_tiles, n_tiles=n_tiles, groups=groups, walk=-(-m_tiles // groups))


WG_PIX, WG_STAGES, WG_MAX_STAGES = 64, 3, 6  # kWgPix, kWgStages, kWgMaxStages (csrc/wgrad_gemm.cuh)


def wgrad_plan(case, sms):
    """plan_wgrad: CTAs per split, 64-pixel blocks, splits, blocks per split, and which limit set the split count"""
    n, h, w, cout = case["gdz"][:4]
    cin, taps = case["gx"][3], case["k"] * case["k"]
    kc_a = 64 if cout >= 64 else (32 if cout >= 32 else 16)
    ma, cout_tiles = -(-min(cout, 128) // kc_a), -(-cout // 128)
    kc_b = 64 if cin % 64 == 0 else (32 if cin % 32 == 0 else 16)
    bn = 128 if cin % 128 == 0 else (64 if cin % 64 == 0 else kc_b)
    nb, cin_tiles = bn // kc_b, cin // bn
    tpc = 1 if (taps == 1 or bn == 128) else 3
    base = cout_tiles * cin_tiles * -(-taps // tpc)
    blocks = _choose_tile(n, h, w, WG_PIX)
    occ_regs = 2 if tpc * bn <= 96 else 1
    stage = WG_PIX * 2 * (kc_a * ma + kc_b * nb * tpc)
    stages = WG_STAGES
    if min(occ_regs, 220 * 1024 // (stage * WG_STAGES + 1024)) <= 1:
        stages = max(WG_STAGES, min(WG_MAX_STAGES, (220 * 1024 - 1024) // stage))
    occ = max(1, min(occ_regs, 220 * 1024 // (stage * stages + 1024)))
    by_occ, by_blocks, by_ws = occ * sms // base, blocks // 8, (128 << 20) // (4 * cout * taps * cin)
    splits = max(1, min(by_occ, by_blocks, by_ws))
    limit = "occupancy" if by_occ <= min(by_blocks, by_ws) else ("blocks / 8" if by_blocks <= by_ws else "workspace")
    bps = -(-blocks // splits)
    splits = -(-blocks // bps)
    return dict(ctas=base, occ=occ, blocks=blocks, splits=splits, bps=bps, last=blocks - (splits - 1) * bps, limit=limit)


# ------------------------------------------------------------------------------------------------------------------------------------
# the recording
# ------------------------------------------------------------------------------------------------------------------------------------
class _Recorder:
    """stands in for the engine's library handle: records every call (entry point, replay case or None, return code) and forwards it"""

    def __init__(self, lib, log):
        self._lib, self.log = lib, log

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("yb200_") or name == "yb200_last_error":
            return fn

        def rec(*a):
            case = _case_of(name, a) if name in GEMMS else None
            rc = fn(*a)
            self.log.append((name, case, rc))
            return rc
        return rec


GEMMS = ("yb200_conv2d_fwd", "yb200_conv2d_fwd_fold", "yb200_conv2d_bn_silu_fwd", "yb200_conv2d_dgrad", "yb200_conv2d_wgrad",
         "yb200_conv2d_wgrad_grouped", "yb200_conv1x1_bias_f32")
# entry points checked by this module, outside the GEMM replays (test that does it)
CHECKED_HERE = {
    "yb200_conv2d_wgrad_workspace": "workspace query: its size is what the recorded wgrad calls were given",
    "yb200_preprocess_focus": "test_focus_and_decode",
    "yb200_yolox_decode": "test_focus_and_decode",
    "yb200_simota_assign": "test_simota_and_losses",
    "yb200_yolox_loss": "test_simota_and_losses",
    "yb200_head_bias_grad": "test_head_bias_grads",
    "yb200_bn_train_apply_silu": "test_batchnorm",
    "yb200_bn_silu_bwd": "test_batchnorm",
    "yb200_bn_param_grads": "test_batchnorm",
    "yb200_bn_eval_affine": "test_eval_batchnorm",
    "yb200_bn_apply_silu": "test_eval_batchnorm",
    "yb200_spp_pool": "test_spp",
    "yb200_spp_pool_bwd": "test_spp",
}
# entry points checked elsewhere at the geometry this plan uses
ELSEWHERE = {
    "yb200_pack_conv_weights_batched": "tests/test_train_bn_gpu.py::test_pack_weights_batched_real_table packs the engine's own layer "
                                       "table, which depends on the layers only, not on the batch or the image size",
}

RECORDING = {}


def _record():
    """one train_step() and one eval_forward() of YoloxEngine(64, 640, 640); the engine is deleted before any replay"""
    from yolov7_d2_b200 import synth
    from yolov7_d2_b200.engine import YoloxEngine

    eng = YoloxEngine(BATCH, SIZE, SIZE)
    names, heads = _yolox_names(eng)
    eng.init_weights(0)
    images, labels = synth.synthetic_batch(BATCH, SIZE, seed=3)
    eng.images_u8.copy_(images.cuda())
    eng.labels.copy_(labels.cuda())
    log = []
    eng.L = _Recorder(eng.L, log)
    try:
        eng.train_step()
        eng.eval_forward()
        torch.cuda.synchronize()
    finally:
        eng.L = eng.L._lib
    layers = [hd.prefix for _, hd in _heads(eng)]
    del eng
    torch.cuda.empty_cache()
    seen, cases = {}, []
    for name, rc_case, _ in log:
        if rc_case is None:
            continue
        label, p, case = rc_case
        key = tuple(sorted(case.items()))
        if key in seen:
            seen[key][1] += 1
            continue
        layer = (heads.get(p) if case["fn"] == "bn_silu" else None) or names.get(p, "?")
        seen[key] = [len(cases), 1]
        cases.append([f"{layer} {label}", case])
    ids = set()
    for i, n in seen.values():
        tid = cases[i][0] + (f" (+{n - 1} more)" if n > 1 else "")
        while tid in ids:
            tid += "'"
        ids.add(tid)
        cases[i][0] = tid
    RECORDING.update(log=[(name, rc) for name, _, rc in log], cases=[tuple(c) for c in cases], layers=layers)


def _recording():
    if not RECORDING and torch.cuda.is_available():
        _record()
    return RECORDING


def _cases(*fns):
    return [(tid, c) for tid, c in _recording().get("cases", []) if c["fn"] in fns]


def _chunk(case):
    """images per chunk of the fp64 references: about 2^26 elements (512 MB) per fp64 tensor of the widest operand"""
    geos = [v for k, v in case.items() if k.startswith("g") and isinstance(v, tuple)]
    per_image = max(g[1] * g[2] * g[4] for g in geos)
    return max(1, (1 << 26) // per_image)


def _kind(c):
    if c["fn"] == "wgrad":
        return "wgrad_grouped" if c["group"] else "wgrad"
    return "fwd_fold" if c["fn"] == "fwd" and c["fold"] else c["fn"]


def pytest_generate_tests(metafunc):
    """the cases are the plan's own calls, recorded when the module is collected on a machine with a GPU"""
    sets = dict(fwd_case=("fwd", "pred"), eval_case=("bn_silu",), dgrad_case=("dgrad",), wgrad_case=("wgrad",),
                probe_wgrad_case=("wgrad",))
    for fixture, fns in sets.items():
        if fixture in metafunc.fixturenames:
            cases = _cases(*fns)
            metafunc.parametrize(fixture, [c for _, c in cases], ids=[t for t, _ in cases])
    if "probe_stats_case" in metafunc.fixturenames:
        cases = [(t, c) for t, c in _cases("fwd") if c["stats"]]
        metafunc.parametrize("probe_stats_case", [c for _, c in cases], ids=[t for t, _ in cases])
    if "layer" in metafunc.fixturenames:
        metafunc.parametrize("layer", _recording().get("layers", []))


def _measured(kind, fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    PEAK[kind] = max(PEAK.get(kind, 0), torch.cuda.max_memory_allocated() - base)


def test_recording_is_complete(cuda):
    """every entry point the step and the inference pass call is checked here or listed with the test that checks it; every call
    succeeded; and the recording reaches the planner branches this module exists for"""
    rec = _recording()
    called = {name for name, _ in rec["log"]}
    unchecked = called - set(GEMMS) - set(CHECKED_HERE) - set(ELSEWHERE)
    assert not unchecked, f"entry points called but neither checked here nor listed: {sorted(unchecked)}"
    failed = [(name, rc) for name, rc in rec["log"] if rc < 0 or (rc != 0 and not name.endswith("_workspace"))]
    assert not failed, failed[:5]
    sms = _sms()
    cases = [c for _, c in rec["cases"]]
    print(f"\n{len(cases)} distinct GEMM geometries recorded on {torch.cuda.get_device_name(0)} ({sms} SMs): "
          + ", ".join(f"{k} {sum(_kind(c) == k for c in cases)}" for k in sorted({_kind(c) for c in cases})))
    print("forward / data gradient: work items, column tiles, CTAs per column tile, most work items per CTA")
    walks = {}
    for tid, c in rec["cases"]:
        if c["fn"] in ("fwd", "dgrad", "bn_silu", "pred"):
            pl = gemm_plan(c, sms)
            walks[tid] = pl
            print(f"  {tid}: BN {pl['bn']} BK {pl['bk']} phases {pl['phases']}: {pl['m_tiles']} x {pl['n_tiles']}, groups {pl['groups']}, "
                  f"walk {pl['walk']}")
    print("weight gradient: CTAs per split, 64-pixel blocks, splits x blocks per split (last split), limit")
    wplans = {}
    for tid, c in rec["cases"]:
        if c["fn"] == "wgrad":
            pl = wgrad_plan(c, sms)
            wplans[tid] = pl
            print(f"  {tid}: {pl['ctas']} CTAs, occupancy {pl['occ']}, {pl['blocks']} blocks = {pl['splits']} x {pl['bps']} "
                  f"(last {pl['last']}), limited by {pl['limit']}")
    fwd = [pl["walk"] for tid, pl in walks.items() if dict(rec["cases"])[tid]["fn"] == "fwd"]
    dg = [(pl["walk"], pl["phases"], pl["groups"]) for tid, pl in walks.items() if dict(rec["cases"])[tid]["fn"] == "dgrad"]
    print(f"largest walk: forward {max(fwd)}, data gradient {max(w for w, _, _ in dg)}")
    assert max(fwd) >= 32, "no forward whose CTAs walk 32 tiles"
    assert max(w for w, _, _ in dg) >= 32, "no data gradient whose CTAs walk 32 tiles"
    assert any(ph == 4 and gr > 1 for _, ph, gr in dg), "no stride-2 four-phase data gradient with groups > 1"
    assert any(pl["limit"] == "occupancy" and pl["last"] < pl["bps"] for pl in wplans.values()), \
        "no weight gradient limited by occupancy with a ragged last split"
    assert any(c["fn"] == "wgrad" and c["group"] for c in cases) and any(c["fn"] == "fwd" and c["fold"] for c in cases)
    assert {"fwd", "bn_silu", "dgrad", "wgrad", "pred"} <= {c["fn"] for c in cases}


# ------------------------------------------------------------------------------------------------------------------------------------
# every distinct GEMM geometry against fp64 (the bound of tests/test_convnext_plan_gpu.py)
# ------------------------------------------------------------------------------------------------------------------------------------
def _replay(kind_case):
    case = dict(kind_case)
    _measured("replay " + _kind(case), lambda: RUN[case.pop("fn")](**case, chunk=_chunk(kind_case)))


def test_fwd(cuda, fwd_case):
    _replay(fwd_case)


def test_eval_fwd(cuda, eval_case):
    _replay(eval_case)


def test_dgrad(cuda, dgrad_case):
    _replay(dgrad_case)


def test_wgrad(cuda, wgrad_case):
    _replay(wgrad_case)


# ------------------------------------------------------------------------------------------------------------------------------------
# exact-integer probes of the pixel-long sums
# ------------------------------------------------------------------------------------------------------------------------------------
def _bits(geo, g, p):
    """bf16 buffer of the view's pitch: inside the view 1 with probability p, else 0; every other channel the sentinel"""
    n, h, w, c, pitch, off = geo
    t = torch.full((n, h, w, pitch), SENTINEL, dtype=torch.bfloat16, device="cuda")
    t[..., off:off + c] = (torch.rand(n, h, w, c, generator=g, device="cuda") < p).to(torch.bfloat16)
    return t


def _exact(what, got, ref):
    got = got.double()
    if not torch.equal(got, ref):
        bad = (got != ref) | ~torch.isfinite(got)
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} values differ from the exact integer result; first at {list(i)}: "
                             f"got {got[i].item():.9g}, exact {ref[i].item():.9g}")


def probe_wgrad(gx, gdz, k, s, cin_real, group, seed=21, chunk=None):
    """yb200_conv2d_wgrad(_grouped) on {0, 1} operands: every weight gradient counts the pixels where both operands are 1 -- an integer
    below 2^20 -- then once more with accumulate = 1 onto integers below 2^10"""
    capi, L = _lib()
    g = _g(seed)
    n, oh, ow, cout = gdz[:4]
    p = min(0.5, math.sqrt(2.0 ** 17 / (n * oh * ow)))  # each count ~2^17 on average
    x, dz = _bits(gx, g, p), _bits(gdz, g, p)
    cin = gx[3]
    xa, dza = _act(capi, x, gx), _act(capi, dz, gdz)
    ws_bytes = L.yb200_conv2d_wgrad_workspace(ctypes.byref(xa), ctypes.byref(dza), k, s)
    assert ws_bytes > 0, L.yb200_last_error()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    shape = (cout, cin_real, k, k)
    ref = wgrad_ref(_sl(x, gx).double(), _sl(dz, gdz).double(), k, s, chunk)[0][:, :cin_real]
    m = _fold_mask(cout, cin, group)[:, :cin_real].bool() if group else torch.ones(shape, dtype=torch.bool, device="cuda")
    g0 = torch.randint(0, 1024, shape, generator=g, device="cuda").float()
    assert float(ref.max()) + 1024 < EXACT_LIMIT and float(ref[m].min()) > 0
    for acc in (0, 1):
        buf, grad = _guarded(shape, g0 if acc else float("nan"))
        if group:
            rc = L.yb200_conv2d_wgrad_grouped(ctypes.byref(xa), ctypes.byref(dza), k, s, cin_real, group, capi.ptr(grad), acc, capi.ptr(ws),
                                              ctypes.c_int64(ws_bytes), capi.stream_ptr())
        else:
            rc = L.yb200_conv2d_wgrad(ctypes.byref(xa), ctypes.byref(dza), k, s, cin_real, capi.ptr(grad), acc, capi.ptr(ws), ctypes.c_int64(ws_bytes),
                                      capi.stream_ptr())
        capi.check(rc, "conv2d_wgrad")
        exp = ref + g0.double() if acc else ref
        _exact(f"weight gradient (accumulate {acc})", grad[m], exp[m])
        _guard_ok(buf, math.prod(shape), "grad")


def _ones_weights(capi, L, cout, cin, k, g, mask, per_row=4):
    """weights with `per_row` ones per output channel at random allowed positions, zeros elsewhere; fp64 copy and packed forward form"""
    score = torch.rand(cout, cin * k * k, generator=g, device="cuda")
    if mask is not None:
        score = score.masked_fill(~mask.reshape(cout, -1).bool(), -1.0)
    w = torch.zeros(cout, cin * k * k, device="cuda")
    w.scatter_(1, score.topk(per_row, 1).indices, 1.0)
    w = w.view(cout, cin, k, k)
    wf = torch.empty(cout, k * k, cin, dtype=torch.bfloat16, device="cuda")
    capi.check(L.yb200_pack_conv_weight(capi.ptr(w), cout, cin, k, cout, cin, capi.ptr(wf), None, capi.stream_ptr()), "pack")
    return w.double(), wf


def probe_stats(gx, gz, k, s, fold, seed=22, chunk=None):
    """yb200_conv2d_fwd(_fold) with BatchNorm statistics on {0, 1} activations and four unit weights per output channel: z is an
    integer in [0, 4] (exact in fp16), and the statistics are integer sums below 2^20, so z, stat_sum and stat_sq must be exact"""
    capi, L = _lib()
    g = _g(seed)
    cin, cout = gx[3], gz[3]
    nst = fold or cout
    per_stat = gz[0] * gz[1] * gz[2] * (cout // nst)
    x = _bits(gx, g, min(0.5, 2.0 ** 17 / (4 * per_stat)))  # Σz ~2^17 per statistic
    mask = _fold_mask(cout, cin, cout // fold) if fold and k == 3 else None
    w, wf = _ones_weights(capi, L, cout, cin, k, g, mask)
    z, z0 = _out_view(gz, g, torch.float16)
    sb, ssum = _guarded((nst,), 0.0, torch.float64)
    qb, ssq = _guarded((nst,), 0.0, torch.float64)
    xa, za = _act(capi, x, gx), _act(capi, z, gz)
    if fold:
        rc = L.yb200_conv2d_fwd_fold(ctypes.byref(xa), capi.ptr(wf), ctypes.byref(za), k, s, capi.ptr(ssum), capi.ptr(ssq), fold, capi.stream_ptr())
    else:
        rc = L.yb200_conv2d_fwd(ctypes.byref(xa), capi.ptr(wf), ctypes.byref(za), k, s, capi.ptr(ssum), capi.ptr(ssq), capi.stream_ptr())
    capi.check(rc, "conv2d_fwd")
    ref = conv_ref(_sl(x, gx).double(), w, k, s, chunk)[0]
    _exact("z", _sl(z, gz), ref)
    _outside_same(z, z0, gz, "z")
    zd = ref.view(-1, nst)
    rs, rq = zd.sum(0), (zd * zd).sum(0)
    assert float(rq.max()) < EXACT_LIMIT and float(rs.min()) > 0
    _exact("sum of z", ssum, rs)
    _exact("sum of z^2", ssq, rq)
    _guard_ok(sb, nst, "sum of z")
    _guard_ok(qb, nst, "sum of z^2")


def test_probe_wgrad(cuda, probe_wgrad_case):
    c = probe_wgrad_case
    _measured("probe " + _kind(c), lambda: probe_wgrad(c["gx"], c["gdz"], c["k"], c["s"], c["cin_real"], c["group"], chunk=_chunk(c)))


def test_probe_stats(cuda, probe_stats_case):
    c = probe_stats_case
    _measured("probe " + _kind(c), lambda: probe_stats(c["gx"], c["gz"], c["k"], c["s"], c["fold"], chunk=_chunk(c)))


def test_spp(cuda):
    """the plan's SPP: 64 x 20 x 20 x 256 (dark5), random and tied maxima"""
    for ties in (False, True):
        check_spp_pool(cuda, (BATCH, 256, SIZE // 32, SIZE // 32), ties)


# ------------------------------------------------------------------------------------------------------------------------------------
# one real 64 x 640 x 640 step: BatchNorm, bias gradients, SimOTA and losses, Focus, decode, eval-path BatchNorm
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def step(cuda):
    st = build_step(cuda, BATCH, SIZE)
    yield st
    del st["eng"]
    torch.cuda.empty_cache()


def _walk(eng, op):
    """the most 128-pixel tiles one CTA of the layer's training forward walks (the stem: its [n, h, w / 4] grouped form)"""
    xb, zb = op.x.buf, op.z.buf
    g = 4 if (op.first and eng.group4) else 1
    case = dict(fn="fwd", gx=(xb.n, xb.h, xb.w // g, g * op.cin_pad), gz=(zb.n, zb.h, zb.w // g, g * op.cout))
    return gemm_plan(case, _sms())["walk"]


def test_batchnorm(step, layer):
    """tests/test_train_bn_gpu.py's checks of one layer: statistics (bound from the per-CTA tile walk of its forward), published
    constants, running statistics, activation, dz and the BatchNorm parameter gradients"""
    _measured("BatchNorm layer", lambda: check_every_batchnorm(step, _walk, layers={layer}))


def test_batchnorm_accumulators_cleared(step):
    eng = step["eng"]
    assert (step["stats"][2 * eng.nbn:] == 0).all(), "the dgamma / dbeta accumulators are not zero after backward"


def test_head_bias_grads(step):
    _check_head_bias(step["eng"], step["grad"], None)


def test_simota_and_losses(step):
    """SimOTA indices bit-exact and the losses to 1e-4 against the oracle on the engine's own head outputs"""
    assert _check_assign_and_losses(step["eng"], step["labels"]) > 0


def test_focus_and_decode(step, cuda):
    """yb200_preprocess_focus exact against oracle.preprocess + focus; yb200_yolox_decode (train and eval) on random raw outputs of the
    plan's [64, 8400, 85] against oracle.decode_train / decode_eval (the tolerance of tests/test_simota_gpu.py::test_decode)"""
    from yolov7_d2_b200 import capi

    eng = step["eng"]
    ref = orc.focus(orc.preprocess(list(step["images"])))
    focus = eng.focus.t.cpu()
    assert torch.equal(focus[..., :12].float(), ref.permute(0, 2, 3, 1)) and (focus[..., 12:] == 0).all(), "Focus output"
    g = torch.Generator().manual_seed(7)
    raw = [torch.randn(BATCH, 85, h, w, generator=g) for h, w, _, _ in eng.levels]
    for eval_mode in (0, 1):
        ref = (orc.decode_eval if eval_mode else orc.decode_train)(raw, [s for _, _, s, _ in eng.levels])
        flat = torch.cat([r.permute(0, 2, 3, 1).reshape(BATCH, -1, 85) for r in raw], 1).contiguous().to(cuda)
        capi.check(eng.L.yb200_yolox_decode(capi.ptr(flat), BATCH, flat.shape[1], 85, eng.lv, len(eng.levels), eval_mode, capi.stream_ptr()),
                   "decode")
        assert torch.allclose(flat.cpu(), ref, rtol=1e-6, atol=1e-6), f"decode (eval {eval_mode})"


def test_eval_batchnorm(step):
    """runs last: eval_forward() replaces the step's BatchNorm constants and activations.  bn_eval_affine: scale = gamma / sqrt(rv + eps),
    shift = beta - rm * scale in fp32 (sqrtf, the division and the additions: at most 8 units of 2^-24 in scale); bn_apply_silu (the layers whose eval BatchNorm is not folded into the
    convolution) against fp64 on the stored z with the published constants, the upsampled copy replicated exactly"""
    eng = step["eng"]
    eng.eval_forward()
    torch.cuda.synchronize()
    for op, hd in _heads(eng):
        name, o, c = hd.prefix, hd.bn_off, hd.c
        gamma, beta = eng.params[name + ".bn.weight"].double(), eng.params[name + ".bn.bias"].double()
        rm, rv = eng.flat_rm[o:o + c].double(), eng.flat_rv[o:o + c].double()
        eps = float(torch.tensor(orc.BN_EPS, dtype=torch.float32))
        s = gamma / torch.sqrt(rv + eps)
        scale, shift = eng.flat_scale[o:o + c].double(), eng.flat_shift[o:o + c].double()
        _fail(name, "eval scale", (scale - s).abs(), 8 * U32 * s.abs())
        _fail(name, "eval shift", (shift - (beta - rm * s)).abs(), 10 * U32 * (rm * s).abs() + U32 * (beta - rm * s).abs())
        if not (any(h.up is not None for h in op.heads) or (op.first and eng.group4)):
            continue  # folded into yb200_conv2d_bn_silu_fwd: replayed by test_eval_fwd
        zb = op.z.buf
        P = zb.n * zb.h * zb.w
        z = zb.view(hd.c0, c).tensor().reshape(P, c).double()
        res = hd.residual.tensor().reshape(P, c).double() if hd.residual is not None else None
        out = hd.out.tensor()
        _check_apply(name, z, eng.flat_scale[o:o + c], eng.flat_shift[o:o + c], out.reshape(P, c), res)
        if hd.up is not None:
            assert torch.equal(hd.up.tensor(), out.repeat_interleave(2, 1).repeat_interleave(2, 2)), f"{name}: upsampled copy"


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst |err| / bound per case class: " + "; ".join(f"{k}: {v:.3g}" for k, v in sorted(WORST.items())))
    if PEAK:
        print("peak device memory per case beyond its inputs: " + "; ".join(f"{k}: {v / 2 ** 30:.2f} GB" for k, v in sorted(PEAK.items())))
