"""The band survey's definition (include/wmbus_b200.h, wmb_set_spectrum) restated in numpy float32, one array operation
per fp32 operation, and the helpers its tests share: the product's records, the restatement's, planted captures."""
import importlib

import numpy as np

BINS = (256, 512, 1024, 2048)


def tables(N):
    """hann[N] and tw[N / 2] = (cos, -sin), computed in double and rounded once"""
    n = np.arange(N, dtype=np.float64)
    hann = (0.5 - 0.5 * np.cos(2.0 * np.pi * n / N)).astype(np.float32)
    k = np.arange(N // 2, dtype=np.float64)
    tw_re = np.cos(2.0 * np.pi * k / N).astype(np.float32)
    tw_im = (-np.sin(2.0 * np.pi * k / N)).astype(np.float32)
    return hann, tw_re, tw_im


def bitrev(N):
    bits = N.bit_length() - 1
    n = np.arange(N)
    r = np.zeros(N, np.int64)
    for b in range(bits):
        r |= ((n >> b) & 1) << (bits - 1 - b)
    return r


def block_power(raw, N):
    """raw: uint8 [nb, 2N] (the blocks' cu8 bytes) -> float32 [nb, N] power per bin, fftshifted"""
    hann, tw_re, tw_im = tables(N)
    u = raw.astype(np.float32)
    i = (u - np.float32(127.5)).astype(np.int32).astype(np.float32)       # (int) truncates toward zero
    xr = i[:, 0::2] * hann
    xi = i[:, 1::2] * hann
    rev = bitrev(N)
    xr, xi = xr[:, rev], xi[:, rev]
    nb = raw.shape[0]
    h = 1
    while h < N:
        xr = xr.reshape(nb, N // (2 * h), 2, h)
        xi = xi.reshape(nb, N // (2 * h), 2, h)
        j = np.arange(h) * (N // (2 * h))
        wr, wi = tw_re[j], tw_im[j]
        ar, ai, br, bi = xr[:, :, 0], xi[:, :, 0], xr[:, :, 1], xi[:, :, 1]
        tr = wr * br - wi * bi
        ti = wr * bi + wi * br
        xr = np.stack([ar + tr, ar - tr], axis=2).reshape(nb, N)
        xi = np.stack([ai + ti, ai - ti], axis=2).reshape(nb, N)
        h *= 2
    p = xr * xr + xi * xi
    return np.roll(p, N // 2, axis=1)


def restated(cu8, N, B, q0=0, d=2, window=(0, 1 << 64), chunk=4096):
    """The records of a run that seeks to IQ sample q0 (0: from the start), pushes cu8 and flushes: (rows as
    (record, start_iq, blocks) tuples, sum [n, N] uint64, peak [n, N] float32).  The flush handles whole 4096-byte
    items only."""
    n_iq = (len(cu8) // 4096) * 2048
    b0, b1 = q0 // N, (q0 + n_iq) // N
    lo, hi = window
    c0 = max(b0, -(-lo * d // N))
    c1 = min(b1, -(-hi * d // N))
    recs = {}
    for a in range(c0, c1, chunk):
        z = min(c1, a + chunk)
        raw = np.asarray(cu8[(a - b0) * 2 * N:(z - b0) * 2 * N]).reshape(z - a, 2 * N)
        p = block_power(raw, N)
        r = np.arange(a, z) // B
        for rec in np.unique(r):
            sel = p[r == rec]
            s = np.rint(sel).astype(np.uint64).sum(axis=0, dtype=np.uint64)
            m = sel.max(axis=0)
            if rec in recs:
                o = recs[rec]
                recs[rec] = (o[0] + s, np.maximum(o[1], m), o[2] + len(sel))
            else:
                recs[rec] = (s, m, len(sel))
    keys = sorted(recs)
    rows = [(int(k), int(k) * B * N, recs[k][2]) for k in keys]
    if not keys:
        return rows, np.zeros((0, N), np.uint64), np.zeros((0, N), np.float32)
    return rows, np.stack([recs[k][0] for k in keys]), np.stack([recs[k][1] for k in keys])


def as_rows(rows):
    return [(int(r["record"]), int(r["start_iq"]), int(r["blocks"])) for r in rows]


def product(pkg, lib, cu8, flags, N, B, pushes=None, seek=None, window=None, take_every=False, **tuning):
    """the product's records for cu8 (pushed whole, or in the given pieces; seek: an IQ position first)"""
    with pkg.WmbusB200(flags, lib=lib, spectrum=(N, B), **tuning) as ctx:
        if seek is not None:
            ctx.seek(seek)
        if window is not None:
            ctx.set_line_window(*window)
        got = []
        if pushes is None:
            ctx.process(cu8.ctypes.data, len(cu8), flush=True)
        else:
            off = 0
            sizes = list(pushes)
            while off < len(cu8):
                n = min(sizes[0] if sizes else len(cu8), len(cu8) - off)
                if sizes:
                    sizes.pop(0)
                ctx.push(cu8.ctypes.data + off, n)
                off += n
                if take_every:
                    got.append(ctx.take_spectrum())
            ctx.poll_flush()
        got.append(ctx.take_spectrum())
        got = [g for g in got if len(g[0])] or got[-1:]
        return (np.concatenate([g[0] for g in got]), np.concatenate([g[1] for g in got]),
                np.concatenate([g[2] for g in got]))


def check_parity(pkg, lib, cu8, flags, N, B, q0=0, d=2, window=None, **kw):
    rows, s, p = product(pkg, lib, cu8, flags, N, B, seek=q0 if q0 else None, window=window, **kw)
    want = restated(cu8, N, B, q0=q0, d=d, window=window or (0, 1 << 64))
    assert_same((rows, s, p), want)
    return rows, s, p


def assert_same(got, want):
    rows, s, p = got
    wr, ws, wp = want
    assert as_rows(rows) == wr, (as_rows(rows)[:5], wr[:5], len(rows), len(wr))
    assert np.array_equal(s, ws), int(np.argwhere(s != ws)[0][0])
    assert np.array_equal(p.view(np.uint32), wp.view(np.uint32)), int(np.argwhere(p.view(np.uint32) != wp.view(np.uint32))[0][0])


def synth_mod():
    return importlib.import_module("rtl-wmbus_b200.synth")


def planted_emitters():
    """a T1, a C1, two S1 emitters spread over a 2.4 MS/s band, at planted offsets (at 40 / 36 their telegrams stand
    about 38 dB above the floor in the peak hold)"""
    E = synth_mod().Emitter
    return [E("T1", 0x71200023, amp=40.0, offset_hz=-600e3, l_field=0x29, period_s=0.11, start_s=0.004, seed=41),
            E("C1A", 0x20338739, amp=40.0, offset_hz=-125e3, l_field=0x19, period_s=0.13, start_s=0.030, seed=42),
            E("S1", 0x19131290, amp=36.0, offset_hz=325e3, l_field=0x19, period_s=0.19, start_s=0.080, seed=43),
            E("S1", 0x02717473, amp=36.0, offset_hz=700e3, l_field=0x19, period_s=0.23, start_s=0.020, seed=44)]


TONE_HZ = -900e3


def planted_capture(emitters, n_bytes=8 << 20, seed=0xB20000A1, tone_amp=30.0):
    """the emitters plus a CW tone at TONE_HZ and noise, 2.4 MS/s (d = 3)"""
    fs = 2.4e6
    buf, plan = synth_mod().synth_capture(n_bytes, fs=fs, emitters=emitters, seed=seed)
    x = buf.numpy().astype(np.float64).reshape(-1, 2)
    if tone_amp:
        ph = 2 * np.pi * TONE_HZ / fs * np.arange(len(x))
        x[:, 0] += tone_amp * np.cos(ph)
        x[:, 1] += tone_amp * np.sin(ph)
    return np.ascontiguousarray(np.clip(np.round(x), 0, 255).astype(np.uint8).reshape(-1)), plan
