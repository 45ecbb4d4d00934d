"""GPU time of the WFM audio bank csdrb_wfm_audio_bank_f_s16 (fractional_decimator_ff 5 | deemphasis_wfm_ff 48000 50e-6 | convert_f_s16 in the
CLI's 1024-sample calls) against the composition it replaces on the same input: the existing fractional decimator bank called on 1024 samples
at a time, the unconsumed rest moved to the front of every row and the bank's state read back after each call, then csdrb_deemphasis_wfm_bank_ff
and csdrb_convert_f_s16 over the decimated rows.  Both give the same bits (checked first).  Workloads: 128 and 1024 channels x 1 s of
discriminator output at 240 kHz (2.4 Msps / 10).  CUDA events around repeated calls after warm-up, at least 1 s per measurement.  Prints one
JSON line with the card name and power limit."""
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import csdr_b200 as cb  # noqa: E402

RATE, TAU, SR, B = 5.0, 50e-6, 48000, 1024


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def timed(fn, min_s=1.0):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    reps, total = 0, 0.0
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    while total < min_s * 1e3:
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        total += t0.elapsed_time(t1); reps += 1
    return total / reps


def workload(channels, n):
    L, s = cb.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cuda").manual_seed(channels)
    t = torch.arange(n, device="cuda", dtype=torch.float32)
    f = torch.rand((channels, 1), generator=g, device="cuda") * 0.05
    x = (0.5 * torch.sin(2 * torch.pi * f * t) + 0.05 * torch.randn((channels, n), generator=g, device="cuda")).contiguous()
    p = cb.WfmAudioParams(RATE, B, TAU, SR)
    consumed = C.c_int(0)
    m = L.csdrb_wfm_audio_bank_outputs(C.byref(p), C.byref(cb.WfmAudioState(0.0, 0)), n, C.byref(consumed))
    out = torch.empty((channels, m), dtype=torch.int16, device="cuda")
    last = torch.zeros(channels, dtype=torch.float32, device="cuda")

    def run_bank():
        last.zero_()
        st = cb.WfmAudioState(0.0, 0)
        rc = L.csdrb_wfm_audio_bank_f_s16(x.data_ptr(), n, channels, n, C.byref(p), C.byref(st), last.data_ptr(), out.data_ptr(), m,
                                          C.byref(consumed), s)
        assert rc == m, L.csdrb_last_error()

    # the composition: one fractional decimator call per 1024 samples (memmove of the rest, state read back), then de-emphasis and s16
    buf = torch.empty((channels, B), dtype=torch.float32, device="cuda")
    cap = int(B / RATE) + 8
    dec_out = torch.empty((channels, cap), dtype=torch.float32, device="cuda")
    dec = torch.empty((channels, m), dtype=torch.float32, device="cuda")
    state = torch.zeros((channels, 3), dtype=torch.int32, device="cuda")
    sb = L.csdrb_fractional_decimator_bank_scratch_bytes(channels, B, RATE)
    scratch = torch.empty(sb + 16, dtype=torch.uint8, device="cuda")
    audio = torch.empty((channels, m), dtype=torch.float32, device="cuda")
    pcm = torch.empty((channels, m), dtype=torch.int16, device="cuda")
    where0 = int(torch.tensor([5.0]).view(torch.int32)[0])

    def run_composition():
        state.zero_(); state[:, 0] = where0
        buf.copy_(x[:, :B])
        pos, k = B, 0
        while True:
            assert L.csdrb_fractional_decimator_bank_ff(buf.data_ptr(), B, dec_out.data_ptr(), cap, channels, B, RATE, 12, None, 0, state.data_ptr(),
                                                        scratch.data_ptr(), sb, s) >= 0
            _, ip, os_ = state[0].tolist()                                  # the read-back: every row consumed the same samples
            dec[:, k:k + os_] = dec_out[:, :os_]
            k += os_
            if pos + ip > n:
                break
            buf[:, :B - ip] = buf[:, ip:].clone()
            buf[:, B - ip:] = x[:, pos:pos + ip]
            pos += ip
        assert k == m
        last.zero_()
        assert L.csdrb_deemphasis_wfm_bank_ff(dec.data_ptr(), m, audio.data_ptr(), m, channels, m, TAU, SR, last.data_ptr(), s) >= 0
        assert L.csdrb_convert_f_s16(audio.data_ptr(), pcm.data_ptr(), channels * m, s) >= 0

    run_bank()
    run_composition()
    same = torch.equal(out, pcm)
    assert same, "the bank and the composition differ"
    t_bank, t_comp = timed(run_bank), timed(run_composition)
    return {"channels": channels, "input_samples_per_channel": n, "audio_samples_per_channel": m, "bits_equal": same, "bank_ms": round(t_bank, 4),
            "composition_ms": round(t_comp, 4), "speedup": round(t_comp / t_bank, 1),
            "bank_channel_seconds_per_s": round(channels * (m / SR) / (t_bank * 1e-3), 1)}


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    res = {"device": card(), "workloads": [workload(128, 240000), workload(1024, 240000)]}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
