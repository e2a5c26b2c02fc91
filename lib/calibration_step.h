/* -*- c++ -*- */
/*
 * calibration_step.h - the armed-calibration step the blocks run at the end of work() (baz_music_doa::calibrate(),
 * baz_music_doa_azel::calibrate()): accumulate the armed items of this call; once all are in, solve for the gains,
 * apply them and record the residual (NaN on failure, with the old gains kept).
 */
#ifndef INCLUDED_BAZ_CALIBRATION_STEP_H
#define INCLUDED_BAZ_CALIBRATION_STEP_H

#include <music_b200.h>

#include <limits>
#include <vector>

inline void calibration_step(music_b200 *h, const float *in, int noutput_items, int &remaining, double az_deg, double el_deg,
                             int kind, double &residual)
{
    if (remaining <= 0) return;
    const int take = noutput_items < remaining ? noutput_items : remaining;
    remaining -= take;
    if (music_b200_calib_accumulate_host(h, in, (uint32_t)take) != MUSIC_B200_OK) {
        remaining = 0;
        residual = std::numeric_limits<double>::quiet_NaN();
        return;
    }
    if (remaining > 0) return;
    std::vector<double> g(2 * MUSIC_B200_MAX_M);
    double stats[2];
    if (music_b200_calib_solve(h, az_deg, el_deg, kind, g.data(), stats) == MUSIC_B200_OK &&
        music_b200_set_calibration(h, g.data()) == MUSIC_B200_OK)
        residual = stats[0];
    else
        residual = std::numeric_limits<double>::quiet_NaN();
}

#endif /* INCLUDED_BAZ_CALIBRATION_STEP_H */
