/*
 * ssb_filter.h -- the sideband filter of `bandpass_fir_fft_cc LO HI 0.05` (README.md:110) on the device, for the programs on the C ABI: csdr-bankd's
 * usb/lsb receive tails and csdr-synth's usb/lsb modulators use the same taps.  Header-only (static), included by each program.
 *
 * Geometry of csdr.c:1822-1831: T = firdes_filter_len(0.05) taps, fft_size N = next_pow2(T), doubled while N - T < 200, input_size N - T + 1; the
 * taps firdes_bandpass_c(T, LO, HI, HAMMING) zero-padded to N and transformed forward (csdr.c:1869), as csdrb_bandpass_fir_fft_bank_cc takes them.
 */
#ifndef CSDR_B200_SSB_FILTER_H
#define CSDR_B200_SSB_FILTER_H

#include <stdlib.h>

#include "csdr_b200.h"

#define SSB_BW 0.05f                                      /* bandpass_fir_fft_cc transition bandwidth of README.md:110 */

/* the N transformed taps in a new device buffer (csdrb_device_free), *fft_size = N and *input_size = N - T + 1; NULL on failure
 * (csdrb_last_error() set, or out of host memory) */
static complexf *ssb_taps_fft(float lo, float hi, int *fft_size, int *input_size, void *stream)
{
    const int T = firdes_filter_len(SSB_BW);
    int N = next_pow2(T);
    if (N - T < 200) N <<= 1;
    complexf *h_taps = calloc((size_t)N, sizeof(complexf));
    complexf *d_taps = csdrb_device_alloc(sizeof(complexf) * (size_t)N), *d_taps_fft = csdrb_device_alloc(sizeof(complexf) * (size_t)N);
    int ok = h_taps && d_taps && d_taps_fft;
    if (ok) {
        firdes_bandpass_c(h_taps, T, lo, hi, WINDOW_HAMMING);
        ok = csdrb_copy_h2d(d_taps, h_taps, sizeof(complexf) * (size_t)N, stream) >= 0 && csdrb_fft_c2c_batch(d_taps, N, d_taps_fft, N, N, 1, 0, stream) >= 0 &&
             csdrb_stream_synchronize(stream) >= 0;
    }
    free(h_taps);
    csdrb_device_free(d_taps);
    if (!ok) { csdrb_device_free(d_taps_fft); return NULL; }
    *fft_size = N; *input_size = N - T + 1;
    return d_taps_fft;
}

#endif
