/* resampler_oracle.c -- TEST INFRASTRUCTURE: a strict-IEEE C restatement of rational_resampler_ff (libcsdr.c:607-636) in the source's
 * loop order, the checker the rational_resampler bank is compared with bit for bit.  Compiled without -ffast-math and without FMA
 * contraction (tests/resampler/resampler.py), so every product and every sum is rounded separately in the order written.
 * One deliberate difference: when no output is possible the reference returns uninitialised fields; this returns {0, 0, last_taps_delay},
 * what the first loop iteration would give. */

/* state[3] = {input_processed, output_size, last_taps_delay} */
void rs_oracle_rational_resampler_ff(const float *input, float *output, int input_size, int interpolation, int decimation, const float *taps,
                                     int taps_length, int last_taps_delay, int *state)
{
    const int output_size = input_size * interpolation / decimation;
    int oi, startingi = 0, delayi = last_taps_delay;
    for (oi = 0; oi < output_size; oi++) {
        float acc = 0;
        startingi = (oi * decimation + interpolation - 1 - last_taps_delay) / interpolation;
        delayi = (last_taps_delay + startingi * interpolation - oi * decimation) % interpolation;
        if (startingi + taps_length / interpolation + 1 > input_size) break;
        for (int i = 0; i < (taps_length - delayi) / interpolation; i++) acc += input[startingi + i] * taps[delayi + i * interpolation];
        output[oi] = acc * interpolation;
    }
    state[0] = startingi;
    state[1] = oi;
    state[2] = delayi;
}

/* The same loop on indices only, for brute-force sweeps: over every call size n = 0..n_max and every last_taps_delay 0..I-1, the number of calls
 * that end on the output cap with input to spare (the loop produced output_size outputs although the next one's filter would still fit the input
 * of the last one: the returned pair is that of the last output, which the next call computes again). */
long rs_oracle_cap_endings(int interpolation, int decimation, int taps_length, int n_max)
{
    long endings = 0;
    for (int input_size = 0; input_size <= n_max; input_size++)
        for (int last_taps_delay = 0; last_taps_delay < interpolation; last_taps_delay++) {
            const int output_size = input_size * interpolation / decimation;
            int oi, startingi = 0;
            for (oi = 0; oi < output_size; oi++) {
                startingi = (oi * decimation + interpolation - 1 - last_taps_delay) / interpolation;
                if (startingi + taps_length / interpolation + 1 > input_size) break;
            }
            if (output_size > 0 && oi == output_size) endings++;
        }
    return endings;
}
