"""Dispatch sweep: every kernel configuration the plan builder gives a generator, SyncNet or discriminator layer at the
batch sizes a user runs, checked layer by layer against float64, at the H100 SXM's 132 SMs, the H100 PCIe's 114 and 66.

make_conv_op / patch_eligible (wav2lip_b200/csrc/host_ops.cuh) pick each layer's box of output pixels from N, halve BN
while the tiles do not fill the SMs, take the channel-major [cm] form when its round fill is close to the row-major
tiles', two M tiles per CTA ([2M]) once there are two rounds of work, and a persistent grid of min(tiles, SMs).  So one
layer runs different code at different N, and a layer can be wrong only in a ragged last box or a partial last round.

Sweep.  The inference plan of every N in 1..128 and every 8th N up to 768 (SWEEP_N: the full range took 10 minutes,
see the table), plus the serving sizes (the benchmark's 640 crops, 1024, SyncNet 256,
the discriminator's 256 x 5 = 1280 frames) is built by a forward on zeros, for the generator (4-D call) in F16, BF16 and
F32X and for SyncNet and the discriminator in F16 and BF16.  Each layer's key (w2l_debug_plan_kernels): kernel family,
BN, BK, MT, [cm], staged epilogue, fold, box width and height, whether the box spans more than one image, patch tile
height, and three edge traits: N % box_n != 0 (ragged last box), a partial last round of the persistent grid, and fewer
tiles than SMs.  The exact box_n is not part of the key: for the 1x1 layers it is min(N, 128), which would make every N
up to 128 a class of its own; the ragged-box trait keeps the case that differs.

Cover.  A greedy set of N reaching every (layer, key) pair of the sweep, always with 640, the stream group's buckets
(powers of two up to its default max_batch of 128), SyncNet 256 and the discriminator at 256 x 5.  At each chosen N the
float64 chain of test_gpu_kernel_parity (_check_chain on the GPU's own exports, reference and bars unchanged; the
generator's fused head too) runs on items 0 and N-1, the first image of every layer's last box and of its last round.
The keys the check ran with must equal the sweep's, and test_every_dispatch_class_is_checked fails on any pair seen and
never checked.  At 114 and 66 SMs (w2l_debug_set_sm_count) only the pairs not already checked at the device's count
need a new N.

Past 2^31.  The generator in F16 at the first N whose largest activation (the 80-channel 96 x 96 input of output_block.0,
from the layer exports) passes 2^31 bytes, and in F32X where its hi + lo planes pass 2^31 elements: the chain on crops on
both sides of the boundary, and those crops bit-identical to the same crops run as a small batch.

Measured on one H100 SXM (80 GB, 700 W, 132 SMs), the file in 8 minutes (sweeps 86 s of it).  Per network and
precision: (layer, key) pairs seen / N values checked (new at the lower counts) / max err/bar over every check:
  case              132 SMs          114 SMs        66 SMs         max err/bar
  generator f16     965 / 74         930 / 10       992 / 37       0.983
  generator bf16    965 / 74         930 / 10       992 / 37       0.998
  generator f32x    996 / 59         953 / 5        981 / 25       0.083
  syncnet f16       527 / 61         497 / 5        538 / 27       0.982
  syncnet bf16      527 / 61         497 / 5        538 / 27       0.997
  disc f16          250 / 55         242 / 6        268 / 22       0.949
  disc bf16         250 / 55         242 / 6        268 / 22       0.992
Past 2^31 at N = 1464 (737280 elements per crop in the largest activation): f16 0.974, f32x 0.074.  A batch of the
boundary crops alone is bit-identical layer by layer up to the first layer whose form differs from N = 1464's
([cm] at face_encoder_blocks.5.0 in f16: 14 layers; all 49 exported layers in f32x).  At 114 SMs every layer keeps
its key at N = 592 (f16, bf16) and 768 (f32x) and the outputs are bit-identical to the device count's; at 66 SMs the
longest such runs are 32 layers (N = 14) and 47 (f32x, N = 1), bit-identical too.  Scaling the [cm] epilogue's shift
by 1 + 2^-10 (one fp16 step) fails the check at every N whose plan has a [cm] layer and at no other.
"""
import ctypes as C
import time

import pytest
import torch

import test_gpu_kernel_parity as P
from oracle import w2l_oracle as O
from test_gpu_kernel_parity import BF16, F16, F32X, PREC_NAME

pytestmark = pytest.mark.gpu

GEN, SYNC, DISC = 0, 1, 2   # NET_GENERATOR, NET_SYNCNET, NET_DISC
NET_NAME = {GEN: "generator", SYNC: "syncnet", DISC: "disc"}
CASES = [(GEN, F16), (GEN, BF16), (GEN, F32X), (SYNC, F16), (SYNC, BF16), (DISC, F16), (DISC, BF16)]
CASE_IDS = [f"{NET_NAME[n]}-{PREC_NAME[p]}" for n, p in CASES]
# every N up to 128 (box_n = min(N, 128) on the 1x1 layers, BN halving and short grids change fastest there), then every
# 8th: the generator's nine sweeps (3 precisions x 3 SM counts) over all of 1..768 took 5.5 minutes, the 21 sweeps of
# this grid take 86 s
SWEEP_N = list(range(1, 129)) + list(range(136, 769, 8))
SERVING = {GEN: [640, 1024], SYNC: [256], DISC: [1280]}
BUCKETS = [1, 2, 4, 8, 16, 32, 64, 128]
ALWAYS = {GEN: [640] + BUCKETS, SYNC: [256], DISC: [1280]}
SM_COUNTS = [0, 114, 66]   # 0: the device's own count
SM_IDS = ["sms-device", "sms-114", "sms-66"]


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in P._CTX.values():
        c.close()
    P._CTX.clear()


def _device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sms(sms):
    if sms > _device_sms():
        pytest.skip(f"the device has {_device_sms()} SMs, fewer than {sms}")
    return sms or _device_sms()


def _layer(k):
    return k["name"].split(" [")[0]


def _work(k):
    return -(-k["m_tiles"] // k["mt"]) * k["n_tiles"]


def _keys(ks, N, S):
    """layer -> dispatch key of one plan of N images built for S SMs."""
    out = {}
    for k in ks:
        w = _work(k)
        out[_layer(k)] = (P._short(k) + ("c" if "[cm]" in k["name"] else ""), k["box_w"], k["box_h"], min(k["box_n"], 2),
                          k["patch_th"], N % k["box_n"] != 0, w % k["grid"] != 0, w < S)
    assert len(out) == len(ks), [k["name"] for k in ks]
    return out


def _items(ks, N):
    """0, N-1, and for every layer the first image of its last box and of its last round (tiles run N-tile fastest,
    then x, y and image)."""
    items = {0, N - 1}
    for k in ks:
        tiles_n = -(-N // k["box_n"])
        items.add((tiles_n - 1) * k["box_n"])
        w = _work(k)
        m = (w - 1) // k["grid"] * k["grid"] // k["n_tiles"] * k["mt"]
        items.add(min(N - 1, m // (k["m_tiles"] // tiles_n) * k["box_n"]))
    return sorted(items)


def _disc_bt(N):
    return (256, 5) if N == 1280 else (N, 1)


# ------------------------------------------------------------------------------------------------------------------
# the sweep: plans built by forwards on zeros, one plan alive at a time
# ------------------------------------------------------------------------------------------------------------------
_SWEEPS = {}


def _zeros_forward(ctx, net, N, z):
    lib = ctx.lib
    p = lambda t: C.c_void_p(t.data_ptr())
    if net == GEN:
        r = lib.w2l_generator_forward(ctx.h, p(z["mel"]), p(z["face"]), p(z["out"]), N, 0, None)
    elif net == SYNC:
        r = lib.w2l_syncnet_forward(ctx.h, p(z["mel"]), p(z["face"]), p(z["a"]), p(z["v"]), N, None)
    else:
        B, T = _disc_bt(N)
        r = lib.w2l_disc_forward(ctx.h, p(z["frames"]), p(z["prob"]), B, T, None)
    from wav2lip_b200 import _lib
    _lib.check(r)


def _sweep(net, prec, sms):
    """N -> (layer -> key, items) over SWEEP_N and the serving sizes."""
    key = (net, prec, sms)
    if key in _SWEEPS:
        return _SWEEPS[key]
    S = _sms(sms)
    ctx = P._ctx(prec)
    ctx.set_debug(False)
    P._load(ctx, net, O.make_state_dict(NET_NAME[net], 0))
    Ns = sorted(set(SWEEP_N + SERVING[net]))
    nmax = max(Ns)
    d = dict(device="cuda", dtype=torch.float32)
    if net == GEN:
        z = {"mel": torch.zeros(nmax, 1, 80, 16, **d), "face": torch.zeros(nmax, 6, 96, 96, **d),
             "out": torch.empty(nmax, 3, 96, 96, **d)}
    elif net == SYNC:
        z = {"mel": torch.zeros(nmax, 1, 80, 16, **d), "face": torch.zeros(nmax, 15, 48, 96, **d),
             "a": torch.empty(nmax, 512, **d), "v": torch.empty(nmax, 512, **d)}
    else:
        z = {"frames": torch.zeros(nmax, 3, 96, 96, **d), "prob": torch.empty(nmax, 1, **d)}
    t0 = time.time()
    rec = {}
    for N in Ns:
        ctx.set_sm_count(sms)   # drops the cached plans
        _zeros_forward(ctx, net, N, z)
        ks = ctx.plan_kernels(net)
        assert all(k["grid"] <= S for k in ks)
        rec[N] = (_keys(ks, N, S), _items(ks, N))
    torch.cuda.synchronize()
    ctx.set_sm_count(0)
    pairs = {(l, k) for keys, _ in rec.values() for l, k in keys.items()}
    print(f"\nREPORT sweep {NET_NAME[net]} {PREC_NAME[prec]} sms={S}: {len(Ns)} plans, {len(pairs)} (layer, key) pairs, "
          f"{time.time() - t0:.1f} s")
    _SWEEPS[key] = rec
    return rec


def _pairs(keys):
    return {(l, k) for l, k in keys.items()}


def _cover(rec, must, done):
    todo = set().union(*(_pairs(k) for k, _ in rec.values())) - done
    chosen = []
    for N in must:
        chosen.append(N)
        todo -= _pairs(rec[N][0])
    while todo:
        N = max(rec, key=lambda n: (len(_pairs(rec[n][0]) & todo), -n))
        chosen.append(N)
        todo -= _pairs(rec[N][0])
    return chosen


# ------------------------------------------------------------------------------------------------------------------
# the float64 chain at one N
# ------------------------------------------------------------------------------------------------------------------
def _check_syncnet_disc(net, prec, N, items):
    from wav2lip_b200 import _lib
    ctx = P._ctx(prec)
    ctx.set_debug(True)
    sd = O.make_state_dict(NET_NAME[net], 0)
    P._load(ctx, net, sd)
    if prec == F16:
        ctx.f16_overflow(clear=True)
    if net == SYNC:
        mel, face = O.make_syncnet_inputs(N, seed=1)
        md, fd = mel.cuda().contiguous(), face.cuda().contiguous()
        a = torch.empty((N, 512), device="cuda")
        v = torch.empty((N, 512), device="cuda")
        _lib.check(ctx.lib.w2l_syncnet_forward(ctx.h, C.c_void_p(md.data_ptr()), C.c_void_p(fd.data_ptr()),
                                               C.c_void_p(a.data_ptr()), C.c_void_p(v.data_ptr()), N, None))
        layers = O.syncnet_layers()
        firsts = {"face_encoder.0": fd[items], "audio_encoder.0": md[items]}
    else:
        B, T = _disc_bt(N)
        frames = O.make_disc_inputs(B, T, seed=1).cuda().contiguous()
        prob = torch.empty((N, 1), device="cuda")
        _lib.check(ctx.lib.w2l_disc_forward(ctx.h, C.c_void_p(frames.data_ptr()), C.c_void_p(prob.data_ptr()), B, T, None))
        layers = O.disc_layers()
        firsts = {"face_encoder_blocks.0.0": torch.cat([frames[:, :, i] for i in range(T)], 0)[:, :, 48:][items]}
    torch.cuda.synchronize()
    if prec == F16:
        assert not ctx.f16_overflow(clear=True)
    names = [n for n, _ in layers]

    def inputs(name, outs):
        return firsts[name] if name in firsts else outs[names[names.index(name) - 1]]
    outs, worst = P._check_chain(ctx, net, layers, sd, inputs, prec, items, f"{NET_NAME[net]} N={N}", trim=True)
    assert sum(o is not None for o in outs.values()) >= len(layers) - 1
    return ctx.plan_kernels(net), worst


def _check_at(net, prec, sms, N, items):
    """Runs the chain at N with the SM count set; returns (kernel rows, max err/bar)."""
    P._ctx(prec).set_sm_count(sms)
    if net == GEN:
        _out, ks, worst = P._run_generator(prec, (), N, items, trim=True)
    else:
        ks, worst = _check_syncnet_disc(net, prec, N, items)
    return ks, worst


_CHECKED = {}   # (net, prec, sms) -> set of (layer, key) checked at that count


def _run_cover(net, prec, sms):
    key = (net, prec, sms)
    if key in _CHECKED:
        return _CHECKED[key]
    S = _sms(sms)
    rec = _sweep(net, prec, sms)
    done = set()
    for lower in SM_COUNTS[:SM_COUNTS.index(sms)]:
        if lower == 0 or lower <= _device_sms():
            done |= _run_cover(net, prec, lower)
    must = ALWAYS[net] if sms == 0 else []
    chosen = _cover(rec, must, done)
    t0 = time.time()
    checked = set()
    for N in chosen:
        keys, items = rec[N]
        ks, worst = _check_at(net, prec, sms, N, items)
        got = _keys(ks, N, S)
        assert got == keys, f"N={N}: the checked plan's dispatch differs from the sweep's: " \
                            f"{[(l, keys.get(l), got[l]) for l in got if keys.get(l) != got[l]]}"
        checked |= _pairs(got)
        print(f"REPORT check {NET_NAME[net]} {PREC_NAME[prec]} sms={S} N={N} items={items}: max err/bar {worst:.3f}")
    P._ctx(prec).set_sm_count(0)
    print(f"REPORT cover {NET_NAME[net]} {PREC_NAME[prec]} sms={S}: N = {chosen}, {time.time() - t0:.1f} s")
    _CHECKED[key] = checked | done
    return _CHECKED[key]


# ------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------
def test_set_sm_count_accepts_only_the_device_range():
    from wav2lip_b200 import _lib
    ctx = P._ctx(F16)
    S = _device_sms()
    for bad in (-1, S + 1, 1 << 20):
        assert ctx.lib.w2l_debug_set_sm_count(ctx.h, bad) == _lib.W2L_EINVAL, bad
    for good in (1, S, 0):
        _lib.check(ctx.lib.w2l_debug_set_sm_count(ctx.h, good))
    # a plan built for one SM runs every tile on one CTA: the same output as the device's count (same keys otherwise)
    P._load(ctx, SYNC, O.make_state_dict("syncnet", 0))
    mel, face = (t.cuda().contiguous() for t in O.make_syncnet_inputs(3, seed=4))
    outs = []
    for n in (1, 0):
        ctx.set_sm_count(n)
        a = torch.empty((3, 512), device="cuda")
        v = torch.empty((3, 512), device="cuda")
        _lib.check(ctx.lib.w2l_syncnet_forward(ctx.h, C.c_void_p(mel.data_ptr()), C.c_void_p(face.data_ptr()),
                                               C.c_void_p(a.data_ptr()), C.c_void_p(v.data_ptr()), 3, None))
        torch.cuda.synchronize()
        ks = ctx.plan_kernels(SYNC)
        assert all(k["grid"] == (1 if n == 1 else min(_work(k), S)) for k in ks)
        outs.append((a, v, [(P._short(k), k["box_w"], k["box_h"], k["box_n"]) for k in ks]))
    if outs[0][2] == outs[1][2]:
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("sms", SM_COUNTS, ids=SM_IDS)
@pytest.mark.parametrize("net,prec", CASES, ids=CASE_IDS)
def test_dispatch_cover_matches_float64(net, prec, sms):
    _run_cover(net, prec, sms)


@pytest.mark.parametrize("sms", SM_COUNTS, ids=SM_IDS)
def test_every_dispatch_class_is_checked(sms):
    S = _sms(sms)
    missing, total = [], 0
    for net, prec in CASES:
        seen = set().union(*(_pairs(k) for k, _ in _sweep(net, prec, sms).values()))
        total += len(seen)
        missing += [(NET_NAME[net], PREC_NAME[prec], l, k) for l, k in sorted(seen - _run_cover(net, prec, sms))]
    print(f"\nREPORT coverage sms={S}: {total} (layer, key) pairs seen, {len(missing)} unchecked")
    assert not missing, f"dispatch classes seen in the sweep and never checked against float64: {missing[:20]}"


@pytest.mark.parametrize("sms", [114, 66], ids=["sms-114", "sms-66"])
@pytest.mark.parametrize("prec", [F16, BF16, F32X], ids=["f16", "bf16", "f32x"])
def test_lower_sm_count_is_bit_identical_where_keys_coincide(prec, sms):
    """At the swept N with the longest run of generator layers (table order) whose kernel, box and form coincide at the
    lower count and the device's, those layers' outputs must be bit-identical (only the grid, and with it which CTA runs
    which tile, differs), and the network output too when every layer coincides."""
    from wav2lip_b200 import _lib
    _sms(sms)
    hi, lo = _sweep(GEN, prec, 0), _sweep(GEN, prec, sms)
    names = [n for n, _ in O.generator_layers()]

    def agree(N):
        a, b = hi[N][0], lo[N][0]
        for i, n in enumerate(names):
            if any(a[l][:5] != b[l][:5] for l in a if l.split(".ph")[0] == n):
                return i
        return len(names)
    N = max(SWEEP_N, key=lambda n: (agree(n), n))
    upto = agree(N)
    assert upto > 0
    ctx = P._ctx(prec)
    ctx.set_debug(True)
    P._load(ctx, GEN, O.make_state_dict("generator", 0))
    mel, face = (t.cuda().contiguous() for t in O.make_generator_inputs(N, seed=5))
    ys, grids = [], []
    for n in (sms, 0):
        ctx.set_sm_count(n)
        y = torch.empty((N, 3, 96, 96), device="cuda")
        _lib.check(ctx.lib.w2l_generator_forward(ctx.h, C.c_void_p(mel.data_ptr()), C.c_void_p(face.data_ptr()),
                                                 C.c_void_p(y.data_ptr()), N, 0, None))
        torch.cuda.synchronize()
        grids.append([k["grid"] for k in ctx.plan_kernels(GEN)])
        ys.append([P._export(ctx, GEN, i) for i in range(upto)] + [y])
    ctx.set_sm_count(0)
    for i in range(upto):
        if ys[0][i] is not None:
            assert torch.equal(ys[0][i], ys[1][i]), f"N={N} {names[i]}: {sms} SMs and the device's count differ"
    if upto == len(names):
        assert torch.equal(ys[0][-1], ys[1][-1]), f"N={N}: network outputs differ"
    print(f"\nREPORT bit-identity {PREC_NAME[prec]} sms={sms} N={N}: {upto} of {len(names)} layers coincide and are "
          f"bit-identical; grids of {sum(a != b for a, b in zip(*grids))} of {len(grids[0])} launches differ")


def _largest_activation(ctx):
    """Elements per crop of the generator's largest block input or output, from the exports of the last plan."""
    names = [n for n, _ in O.generator_layers()]
    mel, face = O.make_generator_inputs(1, seed=2)
    layers, inputs = P._generator_inputs(mel, face, F16)
    outs = {n: P._export(ctx, GEN, i) for i, n in enumerate(names)}
    best = 0
    for n in names:
        for t in (outs[n], inputs(n, outs)):
            if t is not None:
                best = max(best, t[0].numel())
    return best


@pytest.mark.parametrize("prec", [F16, F32X], ids=["f16", "f32x"])
def test_generator_past_2_31(prec):
    from wav2lip_b200 import _lib
    ctx = P._ctx(prec)
    ctx.set_sm_count(0)
    # the shapes, and the plan bytes per crop, from keep-all plans of one and two crops
    P._run_generator(prec, (), 1, [0])
    E = _largest_activation(ctx)
    db1 = ctx.device_bytes()
    P._run_generator(prec, (), 2, [0, 1])   # (reloading the weights dropped the plan of one crop)
    per_crop = ctx.device_bytes() - db1
    planes = 2 if prec == F32X else 1
    # F16: bytes (2 per element) pass 2^31; F32X: elements of the hi + lo planes pass 2^31 (and their bytes, earlier)
    b_el = (1 << 31) // (planes * E) if prec == F32X else (1 << 31) // (2 * E)
    N = b_el + 8
    bounds = {b_el} | ({(1 << 31) // (4 * E)} if prec == F32X else set())
    items = sorted({0, N - 1} | {b + d for b in bounds for d in (-1, 0, 1)})
    need = per_crop * N + 4 * E * N + 3 * N * 6 * 9216 * 4 + (4 << 30)
    free, _total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{free / 2**30:.1f} GiB free on the device, this case needs about {need / 2**30:.1f} GiB")
    assert N * E * 2 * planes > (1 << 31) and (N * E * planes > (1 << 31) if prec == F32X else True)
    t0 = time.time()
    out, ks, worst = P._run_generator(prec, (), N, items, trim=True)
    big = {}
    for i in range(len(O.generator_layers())):
        y = P._export(ctx, GEN, i)
        big[i] = None if y is None else y[items]
        del y
    torch.cuda.empty_cache()
    # the same crops as a small batch
    mel, face = O.make_generator_inputs(N, seed=2)
    md, fd = mel[items].cuda().contiguous(), face[items].cuda().contiguous()
    small = torch.empty((len(items), 3, 96, 96), device="cuda")
    _lib.check(ctx.lib.w2l_generator_forward(ctx.h, C.c_void_p(md.data_ptr()), C.c_void_p(fd.data_ptr()),
                                             C.c_void_p(small.data_ptr()), len(items), 0, None))
    torch.cuda.synchronize()
    ks_small = ctx.plan_kernels(GEN)
    form = lambda k: (k["family"], "[cm]" in k["name"], k["fold"], k["head"])
    names = [n for n, _ in O.generator_layers()]
    assert [_layer(k) for k in ks] == [_layer(k) for k in ks_small]
    # table index of the first layer whose arithmetic form differs between the two plans
    diverge = min((names.index(_layer(a).split(".ph")[0]) for a, b in zip(ks, ks_small) if form(a) != form(b)),
                  default=None)
    compared = 0
    for i, n in enumerate(names):
        if diverge is not None and i >= diverge:
            break
        ys = P._export(ctx, GEN, i)
        if ys is None or big[i] is None:
            continue
        assert torch.equal(ys, big[i]), f"{n}: crops {items} differ between N={N} and a batch of {len(items)}"
        compared += 1
    if diverge is None:
        assert torch.equal(small, out[items])
    print(f"\nREPORT past 2^31 {PREC_NAME[prec]}: N={N} largest activation {E} elements/crop "
          f"({N * E * 2 * planes / 2**30:.2f} GiB), items {items}: max err/bar {worst:.3f}, {compared} layers "
          f"bit-identical to a batch of {len(items)}"
          + ("" if diverge is None else f" (forms differ from {names[diverge]})")
          + f", {time.time() - t0:.1f} s")
