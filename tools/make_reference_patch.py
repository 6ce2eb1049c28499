#!/usr/bin/env python
"""Generates integration/reference_b200.patch: the reference-side binding a maintainer applies to
charlie-foxtrot/RTLSDR-Airband to build it WITH_B200 (demodulate_b200() from this repository in place of demodulate()).

The patch is produced mechanically from a pristine reference tree (default /root/reference) so that it always applies:
copies of the touched files are edited by the small, anchored substitutions below and `diff -u` writes the result.  Nothing
else of the reference is reproduced here.  tests/test_reference_binding.py applies the patch to a scratch copy, compiles the
host adapter against the patched headers (third-party headers stubbed by integration/stubs/) and checks the layout facts the
adapter relies on.

    python tools/make_reference_patch.py [--ref /root/reference] [--out integration/reference_b200.patch]
"""
import argparse
import os
import re
import shutil
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = ["src/rtl_airband.h", "src/rtl_airband.cpp", "src/config.cpp", "src/output.cpp", "src/CMakeLists.txt"]


def sub_once(text, old, new, what):
    if text.count(old) != 1:
        raise SystemExit(f"anchor for '{what}' found {text.count(old)} times (expected 1): the reference changed")
    return text.replace(old, new)


def edit_header(t):
    t = sub_once(t, '#include "squelch.h"\n', '#include "squelch.h"\n\n#ifdef WITH_B200\n#include "airband_b200.h"       // C ABI of the GPU demodulation engine\n'
                 '#include "airband_b200_host.h"  // b200_freq_cfg, b200_freq_stats\n#endif /* WITH_B200 */\n', "engine headers")
    t = sub_once(t, "    enum modulations modulation;\n};\n", "    enum modulations modulation;\n#ifdef WITH_B200\n    b200_freq_cfg b200_cfg;      // what config.cpp handed to squelch / notch_filter / lowpass_filter\n"
                 "    b200_freq_stats b200_stats;  // Squelch read-outs refreshed from the engine\n#endif /* WITH_B200 */\n};\n", "freq_t fields")
    t = sub_once(t, "extern mixer_t* mixers;\n", "extern mixer_t* mixers;\n#ifdef WITH_B200\nextern int devices_running;\nextern \"C\" int b200_fm_demod(void);\n"
                 "extern \"C\" void* demodulate_b200(void* params);  // drop-in for demodulate()\nextern \"C\" int b200_mixer_is_gpu(const mixer_t* m);\n#endif /* WITH_B200 */\n", "externs")
    return t


def edit_main(t):
    t = sub_once(t, "static int devices_running = 0;\n", "#ifdef WITH_B200\nint devices_running = 0;  // read by demodulate_b200()\n#else\nstatic int devices_running = 0;\n#endif /* WITH_B200 */\n",
                 "devices_running")
    t = sub_once(t, "enum fm_demod_algo fm_demod = FM_FAST_ATAN2;\n", "enum fm_demod_algo fm_demod = FM_FAST_ATAN2;\n#ifdef WITH_B200\nextern \"C\" int b200_fm_demod(void) {\n    return fm_demod == FM_QUADRI_DEMOD ? 1 : 0;\n}\n#endif /* WITH_B200 */\n",
                 "fm_demod accessor")
    t = sub_once(t, "        pthread_create(&demod_threads[i], NULL, &demodulate, &demod_params[i]);\n",
                 "#ifdef WITH_B200\n        pthread_create(&demod_threads[i], NULL, &demodulate_b200, &demod_params[i]);\n#else\n"
                 "        pthread_create(&demod_threads[i], NULL, &demodulate, &demod_params[i]);\n#endif /* WITH_B200 */\n", "thread start")
    return t


def edit_config(t):
    t = sub_once(t, "static struct freq_t* mk_freqlist(int n) {\n",
                 "#ifdef WITH_B200\n#define B200_CFG(fr, field, v) ((fr).b200_cfg.field = (v))\n#else\n#define B200_CFG(fr, field, v) ((void)0)\n#endif /* WITH_B200 */\n\n"
                 "static struct freq_t* mk_freqlist(int n) {\n", "macro")
    t = sub_once(t, "        fl[i].modulation = MOD_AM;\n", "        fl[i].modulation = MOD_AM;\n        B200_CFG(fl[i], squelch_snr_db, -1.0f);  // not set\n", "mk_freqlist default")
    rules = [
        (r"^(\s*)channel->freqlist\[f\]\.squelch\.set_squelch_level_threshold\((.+)\);\n", r"\g<0>\1B200_CFG(channel->freqlist[f], squelch_level, \2);\n", 3),
        (r"^(\s*)channel->freqlist\[f\]\.squelch\.set_squelch_snr_threshold\((.+)\);\n", r"\g<0>\1B200_CFG(channel->freqlist[f], squelch_snr_db, \2);\n", 2),
        (r"^(\s*)channel->freqlist\[f\]\.notch_filter = NotchFilter\(freq, WAVE_RATE, q\);\n",
         r"\g<0>\1B200_CFG(channel->freqlist[f], notch_hz, freq);\n\1B200_CFG(channel->freqlist[f], notch_q, q);\n", 2),
        (r"^(\s*)channel->freqlist\[f\]\.squelch\.set_ctcss_freq\(freq, WAVE_RATE\);\n", r"\g<0>\1B200_CFG(channel->freqlist[f], ctcss_hz, freq);\n", 2),
        (r"^(\s*)channel->freqlist\[f\]\.lowpass_filter = LowpassFilter\(\(float\)bandwidth / 2, WAVE_RATE\);\n",
         r"\g<0>\1B200_CFG(channel->freqlist[f], lowpass_hz, (float)bandwidth / 2);\n", 2),
    ]
    for pat, rep, want in rules:
        t, n = re.subn(pat, rep, t, flags=re.M)
        if n != want:
            raise SystemExit(f"config.cpp: pattern {pat!r} matched {n} times (expected {want}): the reference changed")
    return t


def edit_output(t):
    t = sub_once(t, "static void print_channel_metric(", "#ifdef WITH_B200\n#define B200_SQ(fr, what) ((fr).b200_stats.what)\n#else\n#define B200_SQ(fr, what) ((fr).squelch.what())\n#endif /* WITH_B200 */\n\n"
                 "static void print_channel_metric(", "stats macro")
    t, n = re.subn(r"channel->freqlist\[k\]\.squelch\.(noise_level|signal_level|squelch_level|open_count|flappy_count|ctcss_count|no_ctcss_count)\(\)",
                   r"B200_SQ(channel->freqlist[k], \1)", t)
    if n != 9:
        raise SystemExit(f"output.cpp: {n} Squelch getters rewritten (expected 9): the reference changed")
    t = sub_once(t, "            mixer_data* mdata = (mixer_data*)(channel->outputs[k].data);\n",
                 "            mixer_data* mdata = (mixer_data*)(channel->outputs[k].data);\n#ifdef WITH_B200\n            if (b200_mixer_is_gpu(mdata->mixer))\n"
                 "                continue;  // summed on the GPU, delivered into mixer->channel by demodulate_b200()\n#endif /* WITH_B200 */\n", "O_MIXER skip")
    return t


def edit_cmake(t):
    anchor = "if(NOT BCM_VC_FOUND)\n\tpkg_check_modules(FFTW3F REQUIRED fftw3f)"
    if t.count(anchor) != 1:
        raise SystemExit("CMakeLists.txt: anchor not found")
    add = ('option(WITH_B200 "Demodulate on an NVIDIA H100 through libairband_b200 (github: airband-b200)" OFF)\n'
           "if(WITH_B200)\n"
           '\tset(B200_ROOT "" CACHE PATH "checkout of the airband-b200 repository (include/, rtlsdr-airband_b200/)")\n'
           "\tadd_definitions(-DWITH_B200 -DABG_WITH_REFERENCE_HEADERS)\n"
           "\tinclude_directories(${B200_ROOT}/include ${B200_ROOT}/rtlsdr-airband_b200/host)\n"
           "\tlist(APPEND rtl_airband_extra_sources ${B200_ROOT}/rtlsdr-airband_b200/host/demod_adapter.cpp)\n"
           "\tlist(APPEND rtl_airband_extra_libs ${B200_ROOT}/rtlsdr-airband_b200/libairband_b200.so)\n"
           "endif()\n\n")
    return t.replace(anchor, add + anchor)


EDITS = {"src/rtl_airband.h": edit_header, "src/rtl_airband.cpp": edit_main, "src/config.cpp": edit_config, "src/output.cpp": edit_output,
         "src/CMakeLists.txt": edit_cmake}


def build_patch(ref: str) -> str:
    tmp = tempfile.mkdtemp(prefix="b200patch_")
    try:
        out = []
        for rel in FILES:
            a = os.path.join(tmp, "a", rel)
            b = os.path.join(tmp, "b", rel)
            os.makedirs(os.path.dirname(a), exist_ok=True)
            os.makedirs(os.path.dirname(b), exist_ok=True)
            shutil.copy(os.path.join(ref, rel), a)
            open(b, "w").write(EDITS[rel](open(a).read()))
            r = subprocess.run(["diff", "-u", "--label", "a/" + rel, "--label", "b/" + rel, a, b], capture_output=True, text=True)
            if r.returncode not in (0, 1):
                raise SystemExit(r.stderr)
            out.append(r.stdout)
        return "".join(out)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    ap.add_argument("--out", default=os.path.join(ROOT, "integration", "reference_b200.patch"))
    args = ap.parse_args()
    patch = build_patch(args.ref)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    open(args.out, "w").write(patch)
    print(f"{args.out}: {patch.count(chr(10))} lines, {patch.count('@@ -') } hunks")


if __name__ == "__main__":
    main()
