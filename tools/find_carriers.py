"""Carriers worth decoding in a capture, from the CLI's band survey (WMBUS_B200_SPECTRUM=<path>): the same finder as
shard.find_carriers(), on the file's mean and peak lines.
    python tools/find_carriers.py <spectrum file>
prints one line per carrier (offset from the capture's centre, on the 25 kHz grid) and per tone, then the
shard.decode_carriers() call that decodes them: the CLI listens at 0 or +-325 kHz only, so carriers elsewhere are
decoded through the Python API, one context per carrier with both chains on it."""
import importlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
shard = importlib.import_module("rtl-wmbus_b200.shard")
pkg = importlib.import_module("rtl-wmbus_b200")


def read_spectrum(path):
    """mean;RECORD;START_IQ_SAMPLE;BLOCKS;HZ_LOW;HZ_STEP;dB... and peak;... lines -> (rows, sum, peak) as
    take_spectrum() returns them (sum rebuilt from the mean: blocks * 10^(dB / 10))"""
    rows, sums, peaks = [], [], []
    with open(path) as f:
        for line in f:
            fld = line.rstrip("\n").split(";")
            if len(fld) < 7:
                continue
            db = np.array([float(x) for x in fld[6:]])
            lin = np.where(np.isneginf(db), 0.0, 10 ** (db / 10))
            if fld[0] == "mean":
                r = np.zeros(1, pkg.spectrum_dtype())
                r["record"], r["start_iq"], r["blocks"] = int(fld[1]), int(fld[2]), int(fld[3])
                r["hz_low"], r["hz_step"], r["bins"] = float(fld[4]), float(fld[5]), len(db)
                rows.append(r)
                sums.append(lin * int(fld[3]))
            elif fld[0] == "peak":
                peaks.append(lin)
    if not rows:
        return np.zeros(0, pkg.spectrum_dtype()), np.zeros((0, 0)), np.zeros((0, 0))
    return np.concatenate(rows), np.array(sums), np.array(peaks)


def main():
    if len(sys.argv) != 2:
        print(__doc__, file=sys.stderr)
        return 1
    rows, s, p = read_spectrum(sys.argv[1])
    if not len(rows):
        print("no records")
        return 0
    fs = -2 * float(rows["hz_low"][0])
    carriers, tones = shard.find_carriers(rows, s, p, fs)
    offs = sorted({off for off, _ in carriers})
    for off in offs:
        print(f"carrier {off:+d} kHz")
    for t in tones:
        print(f"tone {t / 1e3:+.1f} kHz")
    if offs:
        print(f"decode: shard.decode_carriers(make_ctx, run, {carriers!r}, flags='-d {round(fs / 0.8e6)}')")
    else:
        print("no carrier found")
    return 0


if __name__ == "__main__":
    sys.exit(main())
