"""Generate tests/golden/*.json by running the UNMODIFIED reference (oracle/_ref/vdl2_ref_{strict,fast},
built from the reference sources by oracle/Makefile) on the deterministic streams of tests/cases.py, and store the
reference's table literals and struct layouts (reference_checks.json).  Needs the reference source tree:
    python tests/golden/make_golden.py REFERENCE_DIR
"""
import json
import os
import re
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
from oracle import pyoracle as po
from tests import cases


def _ref_frames(c, flavour):
    with tempfile.NamedTemporaryFile(suffix=".iq") as tf:
        tf.write(np.ascontiguousarray(c["iq"]).view(np.uint8).tobytes()); tf.flush()
        fr, _ = po.run_ref(tf.name, po.FMT_S16 if c["fmt"] == "s16" else po.FMT_U8, c["oversample"], c["centerfreq"],
                           c["freqs"], flavour=flavour, chunk=c["chunk"])
    return [dict(channel=f["channel"], idx=f["idx"], hex=f["data"].hex(), synd_weight=f["synd_weight"],
                 datalen_octets=f["datalen_octets"], num_fec_corrections=f["num_fec_corrections"],
                 frame_pwr_dbfs=f["frame_pwr_dbfs"], nf_pwr_dbfs=f["nf_pwr_dbfs"], ppm_error=f["ppm_error"]) for f in fr]


def reference_checks(ref_dir):
    """reference output on the CPU differential streams, the reference's header-FEC / CRC tables and the sizes and
    offsets of the structures include/vdl2_dropin.h mirrors (oracle/layout_check, built against the reference's headers)"""
    out = {}
    for name, c, flavour in (("replicas_strict", cases.case_replicas(n_slots=8, n_rep=2, duration=0.4), "strict"),
                             ("replicas_fast", cases.case_replicas(n_slots=8, n_rep=2, duration=0.4), "fast"),
                             ("stress", cases.case_stress(), "strict"), ("fuzz", cases.case_fuzz(), "strict")):
        out[name] = dict(iq_sha256=cases.iq_sha256(c), flavour=flavour, frames=_ref_frames(c, flavour))
    src = open(os.path.join(ref_dir, "src", "decode.c")).read()
    out["tables"] = dict(
        parity_check_rows=[int(x, 2) for x in re.findall(r"0b([01]{25})", src.split("syndtable")[0])],
        syndrome_patterns=[int(x, 2) for x in re.findall(r"0b([01]{25})", src.split("syndtable")[1].split("synd_weight")[0])],
        synd_weight=[int(x) for x in re.findall(r"\d+", src.split("synd_weight[1<<HDRFECLEN] = {")[1].split("}")[0])],
        crctable=[int(x, 16) for x in re.findall(r"0x([0-9A-F]{4})", open(os.path.join(ref_dir, "src", "crc.c")).read().split("crctable[256]")[1])][:256])
    lines = subprocess.run([os.path.join(os.path.dirname(po.__file__), "_ref", "layout_check")], check=True,
                           capture_output=True, text=True).stdout.splitlines()
    out["layout"] = {m.group(1): int(m.group(2)) for m in (re.match(r"(.+?)\s+reference\s+(\d+)", l) for l in lines) if m}
    with open(os.path.join(cases.GOLDEN, "reference_checks.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("reference_checks: " + ", ".join(f"{k} {len(v['frames'])} frames" for k, v in out.items() if "frames" in v))


def k2_corpus_reference():
    """the reference's own demod() on the decimated samples of the K2 corpus (tests/k2_corpus.py): per channel, the
    number of frames and a digest of their FRAME lines (strict build, oracle/ref_dec_harness.c), on the channels where
    the reference's behaviour is defined"""
    import hashlib
    from tests import k2_corpus as kc
    out = {}
    for name in kc.STAGES:
        s, ok = kc.stage(name), set(kc.reference_defined(name))
        per = {}
        for line in po.run_ref_dec(s["dec"], s["freqs"], s["max_ppm"]):
            if int(line.split()[1][3:]) in ok:
                per.setdefault(int(line.split()[1][3:]), []).append(line)
        out[name] = dict(dec_sha256=hashlib.sha256(s["dec"].tobytes()).hexdigest(), max_ppm=s["max_ppm"],
                         n_frames=sum(len(v) for v in per.values()),
                         channels={str(c): [len(v), hashlib.sha256("\n".join(v).encode()).hexdigest()[:16]] for c, v in sorted(per.items())})
    with open(os.path.join(cases.GOLDEN, "k2_corpus_reference.json"), "w") as f:
        json.dump(out, f, indent=0)
    print("k2_corpus_reference: " + ", ".join(f"{k} {v['n_frames']} frames" for k, v in out.items()))


def main(ref_dir):
    po.build()
    reference_checks(ref_dir)
    k2_corpus_reference()
    for name, fn in cases.ALL_GOLDEN.items():
        c = fn()
        with tempfile.NamedTemporaryFile(suffix=".iq", delete=False) as tf:
            if name == "wav":
                tf.write(c["raw_bytes"])      # the reference feeds the whole file, header included
            else:
                tf.write(np.ascontiguousarray(c["iq"]).view(np.uint8).tobytes())
            path = tf.name
        out = dict(name=name, fs=c["fs"], oversample=c["oversample"], fmt=c["fmt"], centerfreq=c["centerfreq"],
                   freqs=c["freqs"], chunk=c["chunk"], iq_sha256=cases.iq_sha256(c),
                   injected=[[f.hex() for f in b.frames] for b in c["bursts"]])
        for fl in ("strict", "fast"):
            fr, _ = po.run_ref(path, po.FMT_S16 if c["fmt"] == "s16" else po.FMT_U8, c["oversample"], c["centerfreq"],
                               c["freqs"], flavour=fl, chunk=c["chunk"])
            out[fl] = [dict(channel=f["channel"], idx=f["idx"], hex=f["data"].hex(), synd_weight=f["synd_weight"],
                            datalen_octets=f["datalen_octets"], num_fec_corrections=f["num_fec_corrections"],
                            frame_pwr_dbfs=f["frame_pwr_dbfs"], nf_pwr_dbfs=f["nf_pwr_dbfs"], ppm_error=f["ppm_error"]) for f in fr]
        os.unlink(path)
        with open(os.path.join(cases.GOLDEN, f"{name}.json"), "w") as f:
            json.dump(out, f, indent=1)
        same = [x["hex"] for x in out["strict"]] == [x["hex"] for x in out["fast"]]
        ninj = sum(len(b) for b in out["injected"])
        print(f"{name}: strict {len(out['strict'])} frames, fast {len(out['fast'])} frames, injected {ninj}, strict==fast bytes: {same}")


if __name__ == "__main__":
    main(sys.argv[1])
