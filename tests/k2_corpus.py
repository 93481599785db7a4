"""Deterministic corpus of decimated-sample scenarios for the K2 sync walk (k2_sync_slice and its host form).

The walk handles a launch in 12-sample blocks (VDL2_WALK_BLOCK) with a tail of n_dec mod 12 samples, attempts sync
every third sample while searching (SYNC_SKIP), keeps the last 160 phases in a ring (SYNC_BUFLEN) and slices one
symbol every tenth sample once locked.  Whether it is right depends on where a sync, a symbol instant, a header, a
burst end or a noise-floor update falls relative to those grids and to the end of a launch.  Every scenario here is
built at the decimated rate (synth.modulate_burst with up = 10, noise and scaling applied there) and fed to the stage
on LAUNCHES, so that those positions are placed on purpose instead of being left to the traffic:

  * each channel is a base stream delayed by a prefix of k samples: within a coherent warp the 32 lanes carry one
    scenario at k = 0..31, elsewhere the lanes of one warp carry unrelated scenarios (the searching and in-burst
    paths diverge) at random k;
  * back-to-back bursts with the next preamble 0..150 samples after the end of the previous burst;
  * digital silence (exact zeros) long enough for mag_lp to decay into the subnormal range, subnormal and signed-zero
    samples, bursts scaled to component magnitudes on both sides of 1e-18 and 1e18 (the fast hypot's guards), clipped
    bursts;
  * preamble phase noise swept across the sync threshold, frequency offsets that drive the preamble unwrap deep in both
    directions, offsets on both sides of max_ppm (a second stage created with max_ppm != 0);
  * headers that announce no FEC or too long a transmission, and a third stage of maximum-length (2047-octet)
    transmissions.

tests/test_k2_corpus.py checks that the oracle's run of the corpus hits every such cell and that the host build of
the device functions agrees with it; tests/test_gpu_k2_corpus.py runs it through the device."""
import functools
import numpy as np
from dumpvdl2_b200 import synth

DEC_RATE = synth.SYMBOL_RATE * synth.SPS          # 105000 decimated samples per second
CENTER = 136975000
BLOCK, SKIP, SPS, RING = 12, 3, 10, 160
MAX_PREFIX = 48

# launch lengths in decimated samples, repeated: every residue mod 12, the lengths around a block (11-13), around
# K2a's 64-sample time slice (63-65) and around the ring (149, 150, 159-161), runs of launches shorter than 160 (the
# phase history then comes from several earlier launches) and shorter than 64, and long launches
LAUNCHES = (1, 2, 11, 12, 13, 63, 64, 65, 149, 150, 159, 160, 161, 995,
            1, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 63, 65, 150, 2399,
            160, 159, 161, 149, 12, 64, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 34, 35, 46, 47, 59, 71, 598, 359, 1006)

ERR_CRC_BAD, ERR_TOO_LONG, ERR_NO_FEC = 2, 3, 4
# how deep the preamble unwrap must go in each direction (steps of 2 pi): the drift scenarios take it to -7 and +6; the
# automaton's 77 states, up to 15 steps, are checked one by one against the reference's arithmetic in test_hostsim.py
UNWRAP_DEPTH = 6


def launch_bounds(n_dec, launches=LAUNCHES):
    """[(start, length)] of the launches that feed n_dec samples"""
    out, pos, i = [], 0, 0
    while pos < n_dec:
        n = min(launches[i % len(launches)], n_dec - pos)
        out.append((pos, n))
        pos += n
        i += 1
    return out


def _burst(bits, amp=0.3, freq_hz=0.0, phase_noise=0.0, noise_rng=None):
    """complex128 baseband of one burst at the decimated rate"""
    sig, first = synth.modulate_burst(bits, up=SPS)
    sig = sig.astype(np.complex128) * amp
    if freq_hz:
        sig *= np.exp(2j * np.pi * freq_hz / DEC_RATE * np.arange(sig.size))
    if phase_noise:                                # on the ramp and the preamble only
        n = first + 16 * SPS
        sig[:n] *= np.exp(1j * phase_noise * noise_rng.standard_normal(n))
    return sig


def _frames_bits(rng, lo=20, hi=90):
    bits, _ = synth.burst_bits(synth.random_frames(rng, int(rng.integers(1, 3)), lo, hi))
    return bits


def _header_only_bits(rng, datalen_bits):
    """a header announcing datalen_bits (no FEC, or too long) followed by random symbols"""
    hdr = synth.header_word(datalen_bits)
    bits = np.array([(hdr >> (24 - i)) & 1 for i in range(25)] + list(rng.integers(0, 2, 200)), np.uint8)
    bits = np.concatenate([bits, np.zeros(-bits.size % 3, np.uint8)])
    return bits ^ synth.scrambler_sequence(bits.size)


def _max_length_bits(rng):
    """a transmission of 2047 octets (9 RS blocks): frames, then flags up to the length"""
    frames = []
    while True:
        f = synth.random_frames(rng, 1, 200, 240)[0]
        if len(synth.hdlc_payload_bits(frames + [f])) > 16300:
            break
        frames.append(f)
    p = synth.hdlc_payload_bits(frames)
    while len(p) <= 8 * 2046:
        p += "01111110"
    assert 8 * 2046 < len(p) <= 8 * 2047
    bits, info = synth.burst_bits_from_payload(p)
    assert info["datalen_octets"] == 2047 and info["num_blocks"] == 9
    return bits


def _place(x, sig, at):
    n = min(sig.size, x.size - at)
    if n > 0:
        x[at:at + n] += sig[:n]
    return at + sig.size


def _traffic(rng, n, amp=0.3, sigma=0.02, gap=(150, 1200), **kw):
    x = sigma / np.sqrt(2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    at = int(rng.integers(100, 700))
    while at < n - 400:
        at = _place(x, _burst(_frames_bits(rng), amp, **kw), at) + int(rng.integers(*gap))
    return x


def scenario(kind, rng, n, param=0.0):
    """base stream of one scenario, complex128 [n]"""
    if kind == "traffic":
        return _traffic(rng, n)
    if kind == "back_to_back":
        # burst, then the next preamble `param` samples after the receiver has taken the last bit of it (about 150
        # samples before the last symbols, the ramp-down and the pulse tail end), repeated
        x = 0.02 / np.sqrt(2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        at = int(rng.integers(50, 400))
        while at < n - 400:
            at = _place(x, _burst(_frames_bits(rng, 10, 40)), at) - 150 + int(param)
        return x
    if kind == "silence":
        # digital silence: mag_lp decays through the subnormal range before the first burst arrives
        x = np.zeros(n, np.complex128)
        at = _place(x, _burst(_frames_bits(rng), 0.3), 3400 + int(rng.integers(0, 200)))
        _place(x, _burst(_frames_bits(rng), 0.3), at + int(rng.integers(0, 300)))
        return x
    if kind == "subnormal":
        # subnormal and signed-zero samples between bursts
        mag = np.float32(1e-40) * rng.integers(0, 40, n)
        x = mag * rng.choice([-1.0, 1.0], n) + 1j * np.float32(1e-42) * rng.integers(-3, 4, n)
        x[rng.random(n) < 0.2] = complex(-0.0, -0.0)
        at = int(rng.integers(200, 900))
        while at < n - 400:
            at = _place(x, _burst(_frames_bits(rng)), at) + int(rng.integers(300, 900))
        return x
    if kind == "tiny":
        return _traffic(rng, n, amp=3e-18, sigma=2e-19)
    if kind == "huge":
        return _traffic(rng, n, amp=9e17, sigma=6e16)
    if kind == "clipped":
        x = _traffic(rng, n, amp=1.6, sigma=0.05)
        return np.clip(x.real, -1, 1) + 1j * np.clip(x.imag, -1, 1)
    if kind == "phase_noise":
        # preamble phase noise around the level where the sync metric crosses SYNC_THRESHOLD
        return _traffic(rng, n, phase_noise=param, noise_rng=rng, gap=(100, 500))
    if kind == "drift":
        # frequency offset: the preamble error steps across +-pi, the unwrap goes deep
        return _traffic(rng, n, freq_hz=param, gap=(100, 500))
    if kind == "bad_header":
        x = 0.02 / np.sqrt(2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        at = int(rng.integers(100, 600))
        for k in range(8):
            datalen = (8, 16, 0x5000, 0x7FFF)[k % 4] if k % 2 == 0 else None
            bits = _header_only_bits(rng, datalen) if datalen else _frames_bits(rng)
            at = _place(x, _burst(bits), at) + int(rng.integers(0, 200))
            if at > n - 400:
                break
        return x
    if kind == "max_length":
        x = 0.02 / np.sqrt(2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        at = _place(x, _burst(_max_length_bits(rng)), int(rng.integers(100, 400)))
        _place(x, _burst(_frames_bits(rng)), at + 200)
        return x
    raise ValueError(kind)


MIXED_KINDS = ("traffic", "silence", "subnormal", "tiny", "huge", "clipped", "bad_header", "back_to_back",
               "phase_noise", "drift")


def _stage_main(n):
    """(kind, param, seed, prefix) per channel of the main stage"""
    rng = np.random.default_rng(0x4B32)
    chans = []
    # coherent warps: one scenario, prefixes 0..31
    for w, kind in enumerate(("traffic", "traffic", "back_to_back", "silence", "bad_header", "phase_noise", "drift",
                              "clipped")):
        param = {"back_to_back": 37.0, "phase_noise": 0.5, "drift": 1800.0}.get(kind, 0.0)
        for lane in range(32):
            chans.append((kind, param, 1000 + w, lane))
    # sweeps: the gap after a burst, preamble phase noise, frequency offset
    for g in range(160):
        chans.append(("back_to_back", float(min(g, 150)), 2000 + g, int(rng.integers(0, MAX_PREFIX))))
    for k, s in enumerate(np.linspace(0.3, 0.75, 96)):
        chans.append(("phase_noise", float(s), 3000 + k, int(rng.integers(0, MAX_PREFIX))))
    for k, f in enumerate(np.linspace(-4500, 4500, 96)):
        chans.append(("drift", float(f), 4000 + k, int(rng.integers(0, MAX_PREFIX))))
    # mixed warps: unrelated scenarios lane by lane
    while len(chans) < 1280:
        i = len(chans)
        kind = MIXED_KINDS[i % len(MIXED_KINDS)]
        param = {"back_to_back": float(rng.integers(0, 151)), "phase_noise": float(rng.uniform(0.3, 0.7)),
                 "drift": float(rng.uniform(-4000, 4000))}.get(kind, 0.0)
        chans.append((kind, param, 5000 + i, int(rng.integers(0, MAX_PREFIX))))
    return chans


def _stage_ppm():
    rng = np.random.default_rng(0x50504D)
    return [("drift", float(f), 6000 + k, int(rng.integers(0, MAX_PREFIX))) for k, f in enumerate(np.linspace(-1500, 1500, 64))]


def _stage_long():
    return [("max_length", 0.0, 7000 + (lane % 4), lane) for lane in range(32)]


STAGES = {
    # name: (channel list, decimated samples per channel, max_ppm)
    "main": (lambda: _stage_main(8000), 8000, 0.0),
    "ppm": (_stage_ppm, 8000, 5.0),
    "long": (_stage_long, 60000, 0.0),
}


@functools.lru_cache(maxsize=None)
def stage(name):
    """dict(dec=float32 [n][n_ch][2], freqs, max_ppm, kinds, prefixes) of one stage of the corpus"""
    make, n, max_ppm = STAGES[name]
    chans = make()
    dec = np.empty((n, len(chans), 2), np.float32)
    base_cache = {}
    for c, (kind, param, seed, prefix) in enumerate(chans):
        key = (kind, param, seed)
        if key not in base_cache:
            base_cache[key] = scenario(kind, np.random.default_rng(seed), n + MAX_PREFIX, param)
        x = base_cache[key][MAX_PREFIX - prefix:MAX_PREFIX - prefix + n]
        with np.errstate(all="ignore"):
            dec[:, c, 0] = x.real.astype(np.float32)
            dec[:, c, 1] = x.imag.astype(np.float32)
    freqs = [CENTER - 500000 + 25000 * (c % 40) for c in range(len(chans))]
    return dict(dec=dec, freqs=freqs, max_ppm=max_ppm, kinds=[ch[0] for ch in chans], params=[ch[1] for ch in chans],
                prefixes=[ch[3] for ch in chans])


def reference_defined(name):
    """channels on which the reference's demod() is defined: above about 1 kHz of carrier offset a symbol's phase step
    less the preamble's drift estimate can fall below -2 pi, and src/demod.c:264 then indexes graycode[] with a negative
    remainder (the oracle and the kernels wrap it, DESIGN §2)"""
    s = stage(name)
    return [c for c, (k, p) in enumerate(zip(s["kinds"], s["params"])) if not (k == "drift" and abs(p) > 1000.0)]


@functools.lru_cache(maxsize=None)
def oracle(name):
    """the oracle's run of one stage, trace and state tap on"""
    from oracle import pyoracle as po
    s = stage(name)
    o = po.Oracle(DEC_RATE, 1, po.FMT_U8, CENTER, s["freqs"], max_ppm=s["max_ppm"], trace=True, state_tap=True)
    o.process_dec(s["dec"])
    return o


def coverage(name, launches=LAUNCHES):
    """hit count of every cell of the stage's run in the oracle, fed on `launches`: {cell: count}"""
    s, o = stage(name), oracle(name)
    dec = s["dec"]
    n, n_ch = dec.shape[:2]
    st = o.states()
    ring = (st & 0xFF).astype(np.int64)
    sclk = ((st >> 8) & 0xFF).astype(np.uint8).view(np.int8).astype(np.int64)
    idle = ((st >> 17) & 1).astype(bool)
    locked = ((st >> 16) & 1).astype(bool) & ~idle
    sclk = np.where(idle, 0, sclk)
    nfcnt = ((st >> 18) & 0x3FF).astype(np.int64)
    attempt = ~locked & (sclk + 1 >= SKIP)
    # position of every sample in its launch: block offset inside the launch's whole blocks, or place in the tail
    pos, length = np.zeros(n, np.int64), np.zeros(n, np.int64)
    starts = []
    for a, ln in launch_bounds(n, launches):
        pos[a:a + ln] = np.arange(ln)
        length[a:a + ln] = ln
        starts.append(a)
    in_tail = pos >= BLOCK * (length // BLOCK)
    cells = {}

    def hit(cell, k=1):
        cells[cell] = cells.get(cell, 0) + int(k)

    # blocks entered on the searching path: ring position x offset of the first attempt (where the 60 reads and the
    # twelve writes of the block wrap), and nfcnt reaching 1000 on each of the four attempts
    entry = (~in_tail) & (pos % BLOCK == 0)
    fast = entry[:, None] & ~locked & ~idle & (sclk >= 0) & (sclk < SKIP)
    rf, nrf = np.unique(ring[fast] * SKIP + (SKIP - 1) - sclk[fast], return_counts=True)
    for v, k in zip(rf.tolist(), nrf.tolist()):
        hit(("ring_entry", v // SKIP, v % SKIP), k)
    nf = nfcnt[fast]
    for j in range(4):
        hit(("nf_update_attempt", j), np.sum(nf == 999 - j))
    hit(("nf_update_tail",), np.sum(in_tail[:, None] & attempt & (nfcnt == 999)))
    # blocks entered in a burst: every symbol phase
    lk = entry[:, None] & locked
    for c in np.unique(sclk[lk]).tolist():
        hit(("locked_entry_sclk", c), np.sum(sclk[lk] == c))
    # attempts at a local minimum of the metric just above SYNC_THRESHOLD (no sync): pherr[1] in [4, 4.5) and the new
    # metric (pherr[1] of the next sample) above it
    p1 = o.pherr1()
    att = attempt[:-1] & ~locked[1:]
    hit(("metric_minimum_just_above_threshold",), np.sum(att & (p1[:-1] >= 4.0) & (p1[:-1] < 4.5) & (p1[1:] > p1[:-1])))
    # the preamble unwrap of every attempt, replayed from the phases the ring holds (src/demod.c:131-144): how far it
    # goes in each direction, in steps of 2 pi
    pr = np.array([q * np.pi / 4 for q in synth.PREAMBLE_STEPS], np.float64).astype(np.float32)
    with np.errstate(all="ignore"):
        phase = np.arctan2(dec[..., 1].astype(np.float64), dec[..., 0].astype(np.float64)).astype(np.float32)
    for c in range(n_ch):
        srch = ~locked[:, c]
        seq = np.concatenate([np.zeros(RING, np.float32), phase[srch, c]])
        j = RING + np.flatnonzero(attempt[srch, c])                 # the attempts' samples in `seq`
        err = seq[j[:, None] - 150 + 10 * np.arange(16)[None, :]] - pr[None, :]
        step = np.diff(err, axis=1).astype(np.float64)
        depth = np.cumsum(np.where(step > np.pi, -1, np.where(step < -np.pi, 1, 0)), axis=1)
        for ext in (depth.min(axis=1, initial=0), depth.max(axis=1, initial=0)):   # attempts by their deepest value
            for d, k in zip(*np.unique(ext, return_counts=True)):
                hit(("unwrap_depth", int(d)), k)
    # events by position: sync, header, end of the burst (last requested bit, or a header that stops it)
    last_end = {}
    for e in sorted(o.events(), key=lambda e: (e["channel"], e["dec_index"], e["kind"])):
        d, ch = int(e["dec_index"]), e["channel"]
        kind = {1: "sync", 2: "header", 3: "end"}[e["kind"]]
        where = ("tail", int(pos[d] - BLOCK * (length[d] // BLOCK))) if in_tail[d] else ("block", int(pos[d] % BLOCK))
        hit((kind,) + where)
        if pos[d] < 3:
            hit((kind, "launch_start", int(pos[d])))
        if e["kind"] == 1:
            hit(("sync_accepted", e["i"][3]))
            if 3.5 <= e["f"][1] < 4.0:
                hit(("sync_metric_just_below_threshold",))
            if ch in last_end:
                gap = d - last_end[ch]
                if gap < 320:
                    hit(("sync_after_reset", gap // 10))
                    if s["kinds"][ch] == "back_to_back":
                        hit(("back_to_back_gap_synced", int(s["params"][ch])))
            if sum(1 for a in starts if d - 150 < a <= d) >= 2:
                hit(("sync_window_over_3_launches",))
        if e["kind"] == 2 and e["i"][3] != 0:
            hit(("header_status", e["i"][3]))
            last_end[ch] = d
        if e["kind"] == 3:
            last_end[ch] = d
            hit(("burst_blocks", e["i"][1]))
    # values
    mag = np.abs(dec).max(axis=2)
    hit(("zero_samples",), np.sum(mag == 0))
    hit(("subnormal_samples",), np.sum((mag > 0) & (mag < np.finfo(np.float32).tiny)))
    hit(("largest_component_in_[1e-19,1e-18)",), np.sum((mag >= 1e-19) & (mag < 1e-18)))
    hit(("largest_component_in_[1e-18,1e-17)",), np.sum((mag >= 1e-18) & (mag < 1e-17)))
    hit(("largest_component_in_(1e17,1e18]",), np.sum((mag > 1e17) & (mag <= 1e18)))
    hit(("largest_component_in_(1e18,1e19]",), np.sum((mag > 1e18) & (mag <= 1e19)))
    hit(("clipped_samples",), np.sum(mag == 1.0))
    z = np.concatenate([np.zeros((1, n_ch), bool), mag == 0, np.zeros((1, n_ch), bool)])
    runs = [np.diff(np.flatnonzero(np.diff(z[:, c].astype(np.int8)))) for c in range(n_ch) if z[:, c].any()]
    hit(("silence_over_2400_samples",), sum(int(np.any(r[::2] > 2400)) for r in runs))
    return cells


def required_cells(name):
    """the cells every run of the stage must hit"""
    if name == "long":
        return [("burst_blocks", 9)]
    if name == "ppm":
        return [("sync_accepted", 0), ("sync_accepted", 1)]
    req = [("ring_entry", r, f) for r in range(RING) for f in range(SKIP)]
    req += [("nf_update_attempt", j) for j in range(4)] + [("nf_update_tail",)]
    req += [("locked_entry_sclk", c) for c in range(SPS)]
    for kind in ("sync", "header", "end"):
        req += [(kind, "block", b) for b in range(BLOCK)] + [(kind, "tail", t) for t in range(BLOCK - 1)]
        req += [(kind, "launch_start", p) for p in range(3)]
    req += [("sync_after_reset", g) for g in range(15, 32)]
    req += [("back_to_back_gap_synced", g) for g in range(151)]
    req += [("sync_metric_just_below_threshold",), ("metric_minimum_just_above_threshold",), ("sync_window_over_3_launches",)]
    req += [("unwrap_depth", d) for d in range(-UNWRAP_DEPTH, UNWRAP_DEPTH + 1)]
    # every way a header leaves the decoder idle (DEC_IDLE): uncorrectable, too long, no FEC
    req += [("header_status", ERR_CRC_BAD), ("header_status", ERR_TOO_LONG), ("header_status", ERR_NO_FEC)]
    req += [("zero_samples",), ("subnormal_samples",), ("largest_component_in_[1e-19,1e-18)",),
            ("largest_component_in_[1e-18,1e-17)",), ("largest_component_in_(1e17,1e18]",),
            ("largest_component_in_(1e18,1e19]",), ("clipped_samples",), ("silence_over_2400_samples",)]
    return req


# ---- ragged spans: the ragged walk (k2_sync_slice_ragged) numbers each receiver's samples by the count it brought to
# the span, so the tails are per receiver.  The fleet's IQ is synthesised at each receiver's own rate; its span counts
# are planned from the oracle's events so that syncs, headers and burst ends fall into tails of every position.
RAGGED_W = 3001                                   # the largest count of a span
RAGGED_LENGTHS = tuple(range(1, 12)) + tuple(range(149, 162)) + tuple(12 * k + r for k, r in zip(range(3, 15), range(12)))


@functools.lru_cache(maxsize=None)
def ragged_fleet(n_rx=48, seconds=0.2):
    """[dict(centre, freqs, os, fmt, buf)] : receiver r has one channel, oversample 10 cu8 or 20 cs16, bursts back to back
    with gaps of 0-4 ms"""
    out = []
    for r in range(n_rx):
        os_, fmt = ((10, "u8"), (20, "s16"))[r % 2]
        fs = DEC_RATE * os_
        rng = np.random.default_rng(0x52324B + r)
        off = (0.0, 25e3, -37.5e3)[r % 3]
        t, bursts = float(rng.uniform(0.001, 0.006)), []
        while t < seconds - 0.02:
            frames = synth.random_frames(rng, 1, 16, 60)
            bursts.append(synth.BurstSpec(t, off, frames, power_dbfs=-14.0))
            t += synth.burst_duration_s(frames) + float(rng.uniform(0.0, 0.004))
        iq = synth.synth_stream(fs, seconds, bursts, es_n0_db=30, fmt=fmt, seed=0x5232 + r)
        centre = 136100000 + 125000 * r
        out.append(dict(centre=centre, freqs=[centre + int(off)], os=os_, fmt=fmt,
                        buf=np.ascontiguousarray(iq).view(np.uint8).reshape(-1)))
    return out


def ragged_n_dec(x):
    return x["buf"].size // (x["os"] * (4 if x["fmt"] == "s16" else 2))


def ragged_oracles():
    """the oracle's run of every receiver of the ragged fleet, trace on"""
    from oracle import pyoracle as po
    res = []
    for x in ragged_fleet():
        o = po.Oracle(DEC_RATE * x["os"], x["os"], po.FMT_S16 if x["fmt"] == "s16" else po.FMT_U8, x["centre"], x["freqs"],
                      trace=True)
        o.process(x["buf"])
        res.append(o)
    return res


def ragged_counts(n_dec, events, k0):
    """one receiver's span counts: each event (sync, header, burst end) the plan can reach lands in the tail of its span,
    at tail position (k0 + k) mod (tail length) for the k-th one; the spans between take RAGGED_LENGTHS in turn and a
    remainder, so the counts hold every residue mod 12, 1..11 and 149..161"""
    counts, pos, k, fill = [], 0, 0, k0
    for d in sorted({int(e["dec_index"]) for e in events}):
        c = RAGGED_LENGTHS[(k0 + k) % len(RAGGED_LENGTHS)]
        q = c % BLOCK
        if q == 0:
            c += 1 + (k % 11)
            q = c % BLOCK
        start = d - BLOCK * (c // BLOCK) - (k0 + k) % q
        if start < pos:
            continue
        while pos < start:                         # fillers up to the start of the event's span
            f = min(RAGGED_LENGTHS[fill % len(RAGGED_LENGTHS)], start - pos)
            counts.append(f)
            pos += f
            fill += 1
        counts.append(c)
        pos += c
        k += 1
    while pos < n_dec:
        f = min(RAGGED_W, n_dec - pos)
        counts.append(f)
        pos += f
    return counts


def ragged_spans(oracles, n_dec):
    """[span][receiver] counts (0 when a receiver's plan has run out of spans)"""
    per = [ragged_counts(n_dec[r], o.events(), 5 * r) for r, o in enumerate(oracles)]
    n_spans = max(len(c) for c in per)
    return [[c[s] if s < len(c) else 0 for c in per] for s in range(n_spans)]


def ragged_tail_cells(spans, oracles):
    """{(kind, tail position): count} of the fleet's events, and the set of counts the receivers brought"""
    cells, lengths = {}, set()
    for r, o in enumerate(oracles):
        bounds, pos = [], 0
        for c in (s[r] for s in spans):
            if c:
                bounds.append((pos, c))
                lengths.add(c)
            pos += c
        starts = np.array([b[0] for b in bounds])
        for e in o.events():
            d = int(e["dec_index"])
            a, c = bounds[int(np.searchsorted(starts, d, side="right")) - 1]
            p = d - a
            if p >= BLOCK * (c // BLOCK):
                key = ({1: "sync", 2: "header", 3: "end"}[e["kind"]], p - BLOCK * (c // BLOCK))
                cells[key] = cells.get(key, 0) + 1
    return cells, lengths


# ---- deferral edges of the ragged walk: the default walk skips a burst's data symbols and slices them after the walk
# (vdl2_defer), one queued burst per lane.  A second fleet of mostly short one-frame bursts back to back, whose span counts
# are planned from the oracle's burst ends (kind 3, the sample of a burst's last symbol) so that each receiver cycles
# through the cases where deferral can go wrong, offset per receiver so that the lanes of a warp are in different ones.
DEFER_CASES = ("end_on_last_sample",         # a span ends exactly on a burst's last symbol
               "end_on_next_first_sample",   # ... one sample before it: the last symbol is the next span's first sample
               "end_on_last_sample_but_one", # ... one sample after it
               "empty_span_while_open",      # a zero-count span while the burst is open
               "empty_spans_while_open",     # several in a row
               "one_sample_spans_in_data",   # a run of one-sample spans inside the burst's data
               "two_ends_in_a_span",         # a span holding two burst ends: the second finds the queue taken
               "three_ends_in_a_span")       # ... three


@functools.lru_cache(maxsize=None)
def defer_fleet(n_rx=64, seconds=0.25):
    """[dict(centre, freqs, os, fmt, buf)]: receiver r has one channel, oversample 10 cu8 or 20 cs16, one-frame bursts of
    8-24 octets back to back with gaps of 0-50 decimated samples, about one in twelve a long one of 150-250 octets"""
    out = []
    for r in range(n_rx):
        os_, fmt = ((10, "u8"), (20, "s16"))[r % 2]
        rng = np.random.default_rng(0x444546 + r)
        off = (0.0, 25e3, -37.5e3)[r % 3]
        t, bursts = float(rng.uniform(0.0005, 0.003)), []
        while t < seconds - 0.03:
            frames = synth.random_frames(rng, 1, 150, 250) if rng.random() < 1 / 12 else synth.random_frames(rng, 1, 8, 24)
            bursts.append(synth.BurstSpec(t, off, frames, power_dbfs=-14.0))
            t += synth.burst_duration_s(frames) + float(rng.integers(0, 51)) / DEC_RATE
        iq = synth.synth_stream(DEC_RATE * os_, seconds, bursts, es_n0_db=30, fmt=fmt, seed=0x4445 + r)
        centre = 136100000 + 125000 * r
        out.append(dict(centre=centre, freqs=[centre + int(off)], os=os_, fmt=fmt,
                        buf=np.ascontiguousarray(iq).view(np.uint8).reshape(-1)))
    return out


@functools.lru_cache(maxsize=None)
def defer_oracles():
    """the oracle's run of every receiver of the deferral fleet, trace and decimated-sample tap on"""
    from oracle import pyoracle as po
    res = []
    for x in defer_fleet():
        o = po.Oracle(DEC_RATE * x["os"], x["os"], po.FMT_S16 if x["fmt"] == "s16" else po.FMT_U8, x["centre"], x["freqs"],
                      trace=True, dec_tap=True)
        o.process(x["buf"])
        res.append(o)
    return res


def defer_counts(n_dec, ends, k0, width=RAGGED_W):
    """one receiver's span counts: its burst ends take the DEFER_CASES in turn from case k0 on; fillers between them take
    RAGGED_LENGTHS in turn"""
    counts, pos, fill = [], 0, k0

    def fill_to(cut):
        nonlocal pos, fill
        while pos < cut:
            f = min(RAGGED_LENGTHS[fill % len(RAGGED_LENGTHS)], cut - pos)
            counts.append(f)
            pos += f
            fill += 1

    def one_span_to(cut, first_end):
        """fillers, then one span up to cut that holds first_end and the walk after it"""
        nonlocal pos
        start = max(pos, cut - width)
        if start >= first_end:
            return False
        fill_to(start)
        counts.append(cut - pos)
        pos = cut
        return True

    ends = sorted(ends)
    j, case = 0, k0
    while j < len(ends):
        e = ends[j]
        if e < pos + 130:                          # too close to where the plan stands: the next one
            j += 1
            continue
        kind = DEFER_CASES[case % len(DEFER_CASES)]
        used = 1
        if kind == "end_on_last_sample":
            fill_to(e + 1)
        elif kind == "end_on_next_first_sample":
            fill_to(e)
        elif kind == "end_on_last_sample_but_one":
            fill_to(e + 2)
        elif kind in ("empty_span_while_open", "empty_spans_while_open"):
            fill_to(e - 100)
            counts += [0] * (1 if kind == "empty_span_while_open" else 4)
        elif kind == "one_sample_spans_in_data":
            fill_to(e - 60)
            counts += [1] * 12
            pos += 12
        else:
            used = 2 if kind == "two_ends_in_a_span" else 3
            if j + used - 1 >= len(ends) or not one_span_to(ends[j + used - 1] + 5, e):
                j += 1
                continue
        j += used
        case += 1
    while pos < n_dec:
        f = min(width, n_dec - pos)
        counts.append(f)
        pos += f
    return counts


def defer_spans(oracles, n_dec):
    """[span][receiver] counts of the deferral fleet (0 when a receiver's plan has run out of spans)"""
    per = [defer_counts(n_dec[r], [int(e["dec_index"]) for e in o.events() if e["kind"] == 3], 3 * r)
           for r, o in enumerate(oracles)]
    n_spans = max(len(c) for c in per)
    return [[c[s] if s < len(c) else 0 for c in per] for s in range(n_spans)]
