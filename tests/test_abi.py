"""CPU: the C-ABI library loads, exports every symbol include/*.h declares, and refuses to run without a GPU
(no CPU fallback on the demodulator path)."""
import ctypes as C
import os
import re
import numpy as np
import pytest
import dumpvdl2_b200 as vd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    txt = open(os.path.join(ROOT, "include", header)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b((?:vdl2gpu_|process_buf_|vdl2_channel_|sincosf_lut_|input_lpf_|demod_sync_|process_samples|rs_init|rs_verify|decode_vdl2_burst|vdl2gpu_dropin_)\w*)\s*\(", txt)))


@pytest.mark.parametrize("header", ["vdl2gpu.h", "vdl2_dropin.h"])
def test_every_declared_symbol_is_exported(header):
    if not os.path.exists(os.path.join(ROOT, "include", header)):
        pytest.skip(f"{header} not present")
    L = vd.load_library()
    names = _declared(header)
    assert len(names) >= 8
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/{header} but not exported by libvdl2gpu.so"


def test_abi_version_and_struct_sizes():
    L = vd.load_library()
    assert L.vdl2gpu_abi_version() == 2
    from dumpvdl2_b200 import api
    assert C.sizeof(api._Config) == 72 and C.sizeof(api._Stats) == 160 and C.sizeof(api._Event) == 80
    assert C.sizeof(api._Burst) == 48


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(vd.Vdl2GpuError, match="no usable CUDA device"):
        vd.Vdl2Channels(2100000, 20, vd.FMT_U8, 136975000, [136975000 + 25000])
    L = vd.load_library()
    assert L.vdl2gpu_device_count() == 0


def test_product_does_not_reach_into_oracle():
    """The oracle is the checker only: nothing under dumpvdl2_b200/ may import, link or load it."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "dumpvdl2_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".c", ".cpp")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                for token in ("pyoracle", "liboracle", "vdl2_oracle", "libhostsim", "pyhostsim", "from oracle", "import oracle"):
                    assert token not in txt, f"{f} references {token}"
    out = os.popen(f"ldd {vd.LIB_PATH}").read()
    assert "oracle" not in out


def test_bad_config_is_rejected():
    L = vd.load_library()
    from dumpvdl2_b200 import api
    cfg = api._Config()
    h = C.c_void_p()
    assert L.vdl2gpu_create(C.byref(cfg), C.byref(h)) == -1          # VDL2GPU_EINVAL
    f = np.array([136975000], np.uint32)
    cfg.sample_rate, cfg.oversample, cfg.n_channels = 2100000, 10, 1    # rate != 105000 * oversample
    cfg.freqs = f.ctypes.data_as(C.POINTER(C.c_uint32))
    assert L.vdl2gpu_create(C.byref(cfg), C.byref(h)) == -1


def test_raw_frame_record_is_valid_dumpvdl2_protobuf():
    """vdl2gpu_serialize_raw_frame writes the reference's archive record (proto/dumpvdl2.proto:25-48): parse it back
    with the stock protobuf runtime against a descriptor mirroring that .proto."""
    import struct
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    from dumpvdl2_b200 import api
    fd = descriptor_pb2.FileDescriptorProto(name="dumpvdl2.proto", package="dumpvdl2", syntax="proto3")
    md = fd.message_type.add(name="vdl2_msg_metadata")
    T = descriptor_pb2.FieldDescriptorProto
    for num, name, typ in ((1, "station_id", T.TYPE_STRING), (2, "frequency", T.TYPE_UINT32), (3, "synd_weight", T.TYPE_UINT32),
                           (4, "datalen_octets", T.TYPE_UINT32), (5, "frame_pwr_dbfs", T.TYPE_FLOAT), (6, "nf_pwr_dbfs", T.TYPE_FLOAT),
                           (7, "ppm_error", T.TYPE_FLOAT), (8, "version", T.TYPE_INT32), (9, "num_fec_corrections", T.TYPE_INT32),
                           (10, "idx", T.TYPE_INT32)):
        md.field.add(name=name, number=num, type=typ, label=T.LABEL_OPTIONAL)
    ts = md.nested_type.add(name="timestamp")
    ts.field.add(name="tv_sec", number=1, type=T.TYPE_INT64, label=T.LABEL_OPTIONAL)
    ts.field.add(name="tv_usec", number=2, type=T.TYPE_INT64, label=T.LABEL_OPTIONAL)
    md.field.add(name="burst_timestamp", number=11, type=T.TYPE_MESSAGE, label=T.LABEL_OPTIONAL, type_name=".dumpvdl2.vdl2_msg_metadata.timestamp")
    fr = fd.message_type.add(name="raw_avlc_frame")
    fr.field.add(name="metadata", number=1, type=T.TYPE_MESSAGE, label=T.LABEL_OPTIONAL, type_name=".dumpvdl2.vdl2_msg_metadata")
    fr.field.add(name="data", number=2, type=T.TYPE_BYTES, label=T.LABEL_OPTIONAL)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    Raw = message_factory.GetMessageClass(pool.FindMessageTypeByName("dumpvdl2.raw_avlc_frame"))

    f = api.Frame()
    f.channel, f.freq, f.burst_seq, f.idx = 3, 136975000, 7, 1
    f.data = bytes(range(200)) + b"\x3e\xf9"
    f.synd_weight, f.datalen_octets, f.num_fec_corrections = 1, 504, -2
    f.frame_pwr_dbfs, f.nf_pwr_dbfs, f.ppm_error = -9.840581, 1.7991041, -0.070490792
    rec = api.serialize_raw_frame(f, station_id="EPWA-1", timestamp=(1790000000, 123456))
    (n,) = struct.unpack(">H", rec[:2])
    assert n == len(rec)                      # the length counts its own two octets (src/output-file.c:181)
    m = Raw.FromString(rec[2:])
    assert m.data == f.data and m.metadata.station_id == "EPWA-1" and m.metadata.frequency == 136975000
    assert (m.metadata.synd_weight, m.metadata.datalen_octets, m.metadata.version, m.metadata.num_fec_corrections, m.metadata.idx) == (1, 504, 1, -2, 1)
    assert np.float32(m.metadata.frame_pwr_dbfs) == np.float32(-9.840581) and np.float32(m.metadata.ppm_error) == np.float32(-0.070490792)
    assert (m.metadata.burst_timestamp.tv_sec, m.metadata.burst_timestamp.tv_usec) == (1790000000, 123456)
    rec0 = api.serialize_raw_frame(f)         # no station id, zero timestamp: fields with default values are omitted
    assert Raw.FromString(rec0[2:]).metadata.station_id == "" and Raw.FromString(rec0[2:]).metadata.HasField("burst_timestamp")
