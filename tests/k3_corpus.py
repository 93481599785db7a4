"""A deterministic corpus of bursts for the burst decoder (K3), each with the oracle's answer.

Every item is what K2 hands K3 for one burst: the still-scrambled bits after the preamble (header included, nbits of
them), the transmission length from the header, a channel and metadata.  `want` is the oracle's restatement of the data
part of decode_vdl2_burst on the same bits (src/decode.c:259-380): status, frames, FEC correction count and the
per-block RS results.  The host form of K3 (tests/test_hostsim.py) and the kernel itself (tests/test_gpu_burst_decoder.py)
walk the same items.

Categories:
  rs        RS blocks with 0-8 corrupted octets (parity included), single- and multi-block, shortened last blocks with 2
            and 4 FEC octets: correct decodes, failures, miscorrections (classified per block against the clean code word)
  geometry  lengths around the FEC-octet thresholds, multiples of 249, 5-9 blocks, the 2047-octet maximum
  hdlc      crafted HDLC edge payloads, random fuzz transmissions, bursts of hundreds of tiny frames
  truncated nbits shorter than the geometry needs (VDL2_ERR_DATA_TRUNCATED / VDL2_ERR_FEC_TRUNCATED)
  volume    mostly one-block bursts of AVLC frames, enough to take the corpus past two grid-strides of K3
"""
import functools
import numpy as np
from dumpvdl2_b200 import synth
from oracle import pyoracle as po

FLAG = "01111110"
N_CHANNELS = 2048            # the channels the items are spread over
K3_GRID = 132 * 16           # blocks of a K3 launch (vdl2_host.cu): more bursts than this take a second grid-stride
ERR_FEC_BAD, ERR_DATA_TRUNCATED, ERR_FEC_TRUNCATED = 9, 5, 6
GEOMETRY_LENGTHS = [1, 2, 3, 4, 30, 31, 32, 67, 68, 69, 248, 249, 250, 251, 252, 279, 280, 317, 498, 499, 747,
                    1245, 1992, 1993, 1994, 2022, 2023, 2040, 2046, 2047]


def stuffed(octets):
    return "".join(format(b, "08b")[::-1] for b in octets).replace("11111", "111110")


def hdlc_edge_payload(trial):
    """(payload, corrupt) of HDLC edge case `trial` (0..39): repeated / missing flags, aborts (seven ones), frames that
    are not whole octets, back-to-back flags, length cuts, multi-block and short-block bursts, RS errors within and
    beyond capacity."""
    rng = np.random.default_rng(1000 + trial)
    pieces = [FLAG]
    for _ in range(int(rng.integers(1, 5))):
        body = stuffed(rng.integers(0, 256, int(rng.integers(0, 120)), dtype=np.uint8))
        kind = int(rng.integers(0, 10))
        if kind == 0:
            body += "1" * 7                                   # abort sequence
        elif kind == 1:
            body += "010"                                     # not a whole number of octets
        elif kind == 2:
            body = ""                                         # back-to-back flags
        pieces.append(body)
        pieces.append(FLAG * int(rng.integers(1, 3)))
    payload = "".join(pieces)
    if trial % 5 == 0:
        payload = payload[:-int(rng.integers(1, 8))]          # closing flag cut short
    if trial % 7 == 0:
        payload = FLAG + stuffed(rng.integers(0, 256, int(rng.integers(250, 900)), dtype=np.uint8)) + FLAG
    corrupt = []
    nblk = -(-(-(-len(payload) // 8)) // 249)
    for _ in range(int(rng.integers(0, 5))):
        corrupt.append((int(rng.integers(0, nblk)), int(rng.integers(0, 20)), int(rng.integers(1, 256))))
    return payload, corrupt


def geometry_payload(n_octets, seed=5000):
    """(payload, corrupt) of exactly n_octets: one frame padded with flags, a corrupted octet in the first block and,
    when the last block is longer than 2 octets, one in the last."""
    rng = np.random.default_rng(seed + n_octets)
    body = FLAG + stuffed(rng.integers(0, 256, max(0, n_octets - 4), dtype=np.uint8)) + FLAG
    payload = (body + FLAG * 300)[:n_octets * 8]              # pad with flags, cut to the exact transmission length
    nblk = -(-n_octets // 249)
    last_len = n_octets - (nblk - 1) * 249
    corrupt = [(0, int(rng.integers(0, min(249, n_octets))), 0x55)]
    if last_len > 2:
        corrupt.append((nblk - 1, int(rng.integers(0, last_len)), 0xAA))
    return payload, corrupt


def fuzz_payloads():
    """240 random transmissions (any bit length 17..16383, random content with a sprinkling of flags, 0..8 corrupted
    octets anywhere in the transmitted code words): yields (payload, corrupt)."""
    rng = np.random.default_rng(0xF0B8)
    for trial in range(240):
        nbits = int(rng.integers(17, 0x4000)) if trial % 3 else int(rng.integers(17, 700))
        if trial % 2:                                        # well-formed: stuffed frames between flags, cut to nbits
            payload = FLAG
            while len(payload) < nbits:
                payload += stuffed(rng.integers(0, 256, int(rng.integers(0, 300)), dtype=np.uint8)) + FLAG * int(rng.integers(1, 3))
            if trial % 4 == 1:
                payload = payload[:nbits]                    # cut anywhere
            else:
                nbits = len(payload) if len(payload) < 0x4000 else nbits
                payload = payload[:nbits]
        else:                                                # raw noise with a few flags dropped in
            p_one = (0.5, 0.8, 0.65)[(trial // 2) % 3]          # ones-heavy noise: many stuffed zeros, flags and aborts
            bits01 = (rng.random(nbits) < p_one).astype(np.uint8)
            payload = "".join("01"[b] for b in bits01)
            for _ in range(int(rng.integers(0, 6))):
                at = int(rng.integers(0, max(1, nbits - 8)))
                payload = payload[:at] + FLAG + payload[at + 8:]
        n_oct = -(-nbits // 8)
        nblk = -(-n_oct // 249)
        corrupt = [(int(rng.integers(0, nblk)), int(rng.integers(0, 255)), int(rng.integers(1, 256)))
                   for _ in range(int(rng.integers(0, 9)) if trial % 3 == 1 else 0)]
        last_len = n_oct - (nblk - 1) * 249
        corrupt = [(r, c, x) for (r, c, x) in corrupt if not (r == nblk - 1 and last_len <= c < 249)]   # keep to transmitted octets
        yield payload, corrupt


def many_frames_payload(rng, n_frames, longest):
    """up to n_frames frames of 1..longest octets (shorter than an AVLC header) between flags, some separated by several
    flags, as many as fit in the longest transmission"""
    payload = FLAG
    for _ in range(n_frames):
        part = stuffed(rng.integers(0, 256, int(rng.integers(1, longest + 1)), dtype=np.uint8)) + FLAG * (1 + (rng.random() < 0.2))
        if len(payload) + len(part) > 0x3FFF:
            break
        payload += part
    return payload


def _geometry(datalen_bits):
    """(datalen_octets, num_blocks, last_len, fec per block) of src/decode.c:233-245"""
    n_oct = -(-datalen_bits // 8)
    nblk = -(-n_oct // 249)
    last_len = n_oct - (nblk - 1) * 249
    return n_oct, nblk, last_len, [6] * (nblk - 1) + [synth.fec_octets_for(last_len)]


def _decode(bits, nbits, datalen_bits):
    descr = bits[:nbits] ^ synth.scrambler_sequence(nbits)
    st, frames, corr, rs = po.decode_burst_bits(descr[25:], datalen_bits)
    return dict(status=int(st), frames=frames, corr=int(corr), rs=[int(r) for r in rs])


def _rs_outcomes(payload, corrupt, rs):
    """Per block the oracle ran: 'ok' (corrupted, decoded to the clean code word), 'fail' or 'miscorrect' (decoded to
    something else), with the block's FEC octets and whether it is the last."""
    p = payload + "0" * (-len(payload) % 8)
    octets = np.packbits(np.frombuffer(p.encode(), np.uint8) - ord("0"), bitorder="little")
    n_oct, nblk, last_len, nfec = _geometry(len(payload))
    out = []
    for r in range(nblk):
        if rs[r] == -128:
            break
        row = np.zeros(249, np.uint8)
        part = octets[r * 249:(r + 1) * 249]
        row[:part.size] = part
        clean = po.rs_encode(row)
        rx = clean.copy()
        rx[249 + nfec[r]:] = 0
        hits = [(c, x) for (q, c, x) in corrupt if q == r]
        for c, x in hits:
            rx[c] ^= x
        ret, fixed = po.rs_verify(rx, nfec[r])
        assert ret == rs[r], "per-block RS result differs from the burst decoder's"
        if nfec[r] == 0:
            kind = "no_fec"                                  # a last block of 1-2 octets carries no FEC: taken as received
        elif ret < 0:
            kind = "fail"
        elif np.array_equal(fixed[:249], clean[:249]):
            kind = "ok" if hits else "clean"
        else:
            kind = "miscorrect"
        out.append((kind, nfec[r], r == nblk - 1))
    return out


def _rs_payload(rng, shape):
    """one frame between flags, of about the length `shape` picks, and 0-8 corrupted octets per block at distinct
    transmitted positions (data and the block's parity octets)"""
    if shape == 0:
        n_oct = int(rng.integers(200, 249))
    elif shape in (1, 2):
        n_oct = int(rng.integers(3, 31)) if shape == 1 else int(rng.integers(31, 68))
    else:
        last = (int(rng.integers(3, 31)), int(rng.integers(31, 68)), int(rng.integers(68, 250)))[shape - 3]
        n_oct = 249 * int(rng.integers(1, 4)) + last
    payload = FLAG + stuffed(rng.integers(0, 256, max(1, int((n_oct - 2) / 1.04)), dtype=np.uint8)) + FLAG
    _, nblk, last_len, nfec = _geometry(len(payload))
    corrupt = []
    for r in range(nblk):
        cols = list(range(last_len if r == nblk - 1 else 249)) + [249 + k for k in range(nfec[r])]
        n_err = int(rng.integers(0, 9)) if (nblk == 1 or rng.random() < 0.4) else int(rng.integers(0, 4))
        for c in rng.choice(len(cols), size=min(n_err, len(cols)), replace=False):
            corrupt.append((r, cols[int(c)], int(rng.integers(1, 256))))
    return payload, corrupt


@functools.lru_cache(maxsize=None)
def corpus():
    """-> list of items (dicts): kind, bits (uint8 0/1, scrambled), nbits, datalen_bits, channel, syndrome, frame_pwr,
    mag_nf, ppm_error, sync_dec_index, freq, want (the oracle's answer), and for kind 'rs' the per-block outcomes"""
    items = []
    meta = np.random.default_rng(0x4B33)

    def add(kind, payload, corrupt, cut=None, **extra):
        try:
            bits, info = synth.burst_bits_from_payload(payload, corrupt_octets=corrupt)
        except ValueError:                                   # no FEC octets for this length
            return None
        nbits = len(bits) if cut is None else cut
        i = len(items)
        it = dict(kind=kind, bits=bits[:nbits], nbits=nbits, datalen_bits=info["datalen_bits"], channel=(i * 7) % N_CHANNELS,
                  syndrome=(i * 2654435761) & 0xFFFFFFFF, frame_pwr=np.float32(meta.uniform(1e-6, 2.0)),
                  mag_nf=np.float32(meta.uniform(1e-7, 0.1)), ppm_error=np.float32(meta.uniform(-40.0, 40.0)),
                  sync_dec_index=(i << 33) | int(meta.integers(0, 1 << 33)), freq=118000000 + 8333 * i,
                  want=_decode(bits, nbits, info["datalen_bits"]), **extra)
        items.append(it)
        return it

    rng = np.random.default_rng(0x525321)
    for k in range(1500):
        payload, corrupt = _rs_payload(rng, k % 6)
        it = add("rs", payload, corrupt)
        it["blocks"] = _rs_outcomes(payload, corrupt, it["want"]["rs"])
    for n in GEOMETRY_LENGTHS + [997, 1000, 1100, 1244, 1246, 1494, 1495, 1743, 1990, 1991]:
        for seed in (5000, 6000, 7000):
            add("geometry", *geometry_payload(n, seed))
    for trial in range(40):
        add("hdlc_edge", *hdlc_edge_payload(trial), trial=trial)
    for payload, corrupt in fuzz_payloads():
        add("fuzz", payload, corrupt)
    for k in range(24):
        add("many_frames", many_frames_payload(rng, int(rng.integers(130, 1000)), (1, 2, 4, 10)[k % 4]), [])
    src = [it for it in items if it["kind"] in ("rs", "geometry") and it["nbits"] > 60]
    for k in range(240):                                     # cut short: in the data part, or in the FEC part
        it = src[int(rng.integers(0, len(src)))]
        n_oct, nblk, _, nfec = _geometry(it["datalen_bits"])
        lo, hi = (25, 25 + 8 * n_oct) if k % 2 == 0 else (25 + 8 * n_oct, 25 + 8 * (n_oct + sum(nfec)))
        cut = int(rng.integers(lo, hi))
        bits = it["bits"]
        i = len(items)
        items.append(dict(it, kind="truncated", bits=bits[:cut], nbits=cut, channel=(i * 7) % N_CHANNELS,
                          want=_decode(bits, cut, it["datalen_bits"])))
    while len(items) < 6000:                                 # volume: AVLC frames, mostly one block, 0-3 corrupted octets
        frames = synth.random_frames(rng, n_frames=int(rng.integers(1, 4)), lo=11, hi=80)
        payload = synth.hdlc_payload_bits(frames)
        _, nblk, last_len, nfec = _geometry(len(payload))
        corrupt = [(int(rng.integers(0, nblk)), int(rng.integers(0, min(249, last_len))), int(rng.integers(1, 256)))
                   for _ in range(int(rng.integers(0, 4)))]
        add("volume", payload, corrupt)
    return items


def burst_counters(items, n_channels=N_CHANNELS):
    """per-channel counters [n_channels][9] that K3 must add for these items (src/decode.c statsd counters; FCS verdicts
    only for frames of 11 octets or more)"""
    cnt = np.zeros((n_channels, po.NUM_COUNTERS), np.uint64)
    for it in items:
        w, c = it["want"], it["channel"]
        cnt[c, 2] += 1
        cnt[c, 3] += w["status"] != 0
        cnt[c, 4] += sum(r != -128 for r in w["rs"])
        cnt[c, 5] += sum(r >= 0 for r in w["rs"])
        cnt[c, 6] += len(w["frames"])
        for f in w["frames"]:
            if len(f) >= 11:
                cnt[c, 7 if po.crc16(f) == 0xF0B8 else 8] += 1
    return cnt
