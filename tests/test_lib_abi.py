"""CPU-side checks of the product library: it loads, exports every symbol include/airband_b200.h declares, the
Python struct mirrors match the C layouts, and without a GPU it fails loudly (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    L = lib.load()
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
    declared = sorted(set(re.findall(r"ABG_API[^;]*?\b(abg_[a-z_0-9]+)\s*\(", hdr)))
    assert declared, "no ABG_API declarations found"
    assert sorted(lib.SYMBOLS) == declared, "airband_b200.lib.SYMBOLS is out of sync with the header"
    for name in declared:
        assert hasattr(L, name), f"libairband_b200.so does not export {name}"
    assert b"sm_90a" in L.abg_version()


def test_struct_layouts_match_header_order():
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()

    def fields(struct):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            for part in decl.split(","):
                names.append(re.sub(r"\[.*?\]", "", part.strip().split()[-1].lstrip("*")))
        return names

    assert fields("abg_channel_cfg") == [f for f, _ in cm.CChannelCfg._fields_]
    assert fields("abg_device_cfg") == [f for f, _ in cm.CDeviceCfg._fields_]
    assert fields("abg_config") == [f for f, _ in cm.CConfig._fields_]
    assert fields("abg_squelch_stats") == [f for f, _ in cm.CSquelchStats._fields_]
    assert fields("abg_options") == [f for f, _ in lib.COptions._fields_]
    assert fields("abg_mixer_input") == [f for f, _ in lib.CMixerInput._fields_]
    assert C.sizeof(cm.CChannelCfg) == 14 * 4


def test_oracle_and_product_share_the_config_layout():
    oh = open(os.path.join(ROOT, "oracle", "airband_oracle.h")).read()
    ph = open(os.path.join(ROOT, "include", "airband_b200.h")).read()

    def body(text, name):
        b = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S).group(1)
        b = re.sub(r"/\*.*?\*/", "", b, flags=re.S)
        return re.sub(r"\s+", " ", b).replace("abo_", "abg_").strip()

    for s in ("channel_cfg", "device_cfg", "config", "squelch_stats"):
        assert body(oh, "abo_" + s) == body(ph, "abg_" + s)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(lib.AbgError) as ei:
        lib.Engine(wl.cfg1())
    assert ei.value.code == -1 and "no CPU fallback" in str(ei.value)


def test_product_never_touches_the_oracle():
    pkg = os.path.join(ROOT, "rtlsdr-airband_b200")
    for dirpath, _, files in os.walk(pkg):
        if "build" in dirpath:
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".h", ".hpp", "Makefile")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle_py" not in text and "libairband_oracle" not in text and "airband_oracle.h" not in text, os.path.join(dirpath, f)


def test_host_adapter_library_exports():
    from airband_b200 import host
    L = host.load()
    for name in host.HOST_SYMBOLS:
        assert hasattr(L, name), name
