"""Mirror of the reference helper module ``baz.music_doa_helper``
(/root/reference/python/music_doa_helper.py), Python-3 clean.

``calculate_antenna_array_response`` keeps the reference's name, arguments and result (nested
list ``[angular_resolution][len(antenna_array)]`` of complex128).  ``music_doa_helper`` keeps the
constructor signature, the 2- or 3-output port layout (:61-64, :91-96), the banner (:76-83)
and ``set_frequency`` (:100-103).  GNU Radio is not present in this image, so instead of
being a ``gr.hier_block2`` it exposes the wrapped block as ``.impl`` and forwards ``work``;
INTEGRATION.md shows the two-line change that turns it back into a hier block.
"""
from __future__ import annotations

import numpy

from .music_doa import music_doa


def unit_vect(theta):
    return numpy.array([numpy.cos(theta), numpy.sin(theta)])  # :29-30


def calculate_antenna_array_response(antenna_array, angular_resolution, l):
    """/root/reference/python/music_doa_helper.py:32-46: for every grid step the response of
    each element is exp(-j 2 pi <p, u(angle)> / lambda).  Evaluated with the same scalar numpy
    calls (numpy.inner, numpy.cos/sin on Python floats, numpy.exp) as the reference, because
    numpy's vectorised cos/sin and a hand-expanded inner product round differently in the last
    ulp, and an ulp in fp64 can flip the complex64 rounding the block sees."""
    positions = [numpy.asarray(p, dtype=numpy.float64) for p in antenna_array]
    response = []
    for step in range(0, angular_resolution):
        angle = (step * 360.0 / angular_resolution) * (numpy.pi / 180.0)
        u = unit_vect(angle)
        response.append([numpy.exp(-1j * 2.0 * numpy.pi * (numpy.inner(p, u) / l)) for p in positions])
    return response


class music_doa_helper(object):
    def __init__(self, m, n, nsamples, angular_resolution, frequency, array_spacing, antenna_array,
                 output_spectrum=False, device=0, device_table=False, refine=False,
                 estimator="music", loading=0.0):
        self.m = m
        self.n = n
        self.nsamples = nsamples
        self.angular_resolution = angular_resolution
        self.l = 299792458.0 / frequency  # :55
        self.antenna_array = [[array_spacing * x, array_spacing * y] for [x, y] in antenna_array]  # :56
        self.output_spectrum = bool(output_spectrum)
        # extension: device_table=True makes set_frequency() rebuild the table on the GPU
        # (music_b200_set_geometry) instead of the K x M Python loop + re-marshalling; same table, bit for bit
        self.device_table = bool(device_table)
        # extension: refine=True reports off-grid angles (music_b200_set_refine); the block then needs the geometry, so
        # the table is installed with set_array_geometry (bit-identical to the one computed below) here and on retunes
        self.refine = bool(refine)

        if (nsamples % m) != 0:
            raise Exception("nsamples must be multiple of m")  # :58-59

        # port item sizes in bytes, :61-64 / :69
        self.input_item_sizes = [8 * nsamples]
        self.output_item_sizes = [4 * n, 4 * n] + ([4 * angular_resolution] if output_spectrum else [])

        print("MUSIC DOA Helper: M: %d, N: %d, # samples: %d, steps of %f degress, lambda: %f, array: %s" % (
            self.m, self.n, self.nsamples, (360.0 / self.angular_resolution), self.l, str(self.antenna_array)))  # :76

        self.array_response = calculate_antenna_array_response(self.antenna_array, self.angular_resolution, self.l)
        self.impl = music_doa(self.m, self.n, self.nsamples, self.array_response, self.angular_resolution,
                              device=device)  # :89
        # extension: estimator="mvdr" / "bartlett" (music_doa.set_estimator); the default keeps the MUSIC spectrum
        if estimator != "music" or loading != 0.0:
            self.impl.set_estimator(estimator, loading)
        if self.refine:
            self.impl.set_array_geometry(self.antenna_array, self.l)
            self.impl.set_refine(True)

    def set_frequency(self, frequency):
        """:100-103"""
        self.l = 299792458.0 / frequency
        if self.device_table or self.refine:
            self.impl.set_array_geometry(self.antenna_array, self.l)
            self.array_response = None  # lives on the device; impl.array_response_c64() reads it back
            return
        self.array_response = calculate_antenna_array_response(self.antenna_array, self.angular_resolution, self.l)
        self.impl.set_array_response(self.array_response)

    def work(self, noutput_items, input_items, output_items):
        """Forward to the wrapped block: outputs (0) angles, (1) levels, (2) spectrum if enabled."""
        if len(output_items) != len(self.output_item_sizes):
            raise ValueError("helper was built with %d output ports" % len(self.output_item_sizes))
        return self.impl.work(noutput_items, input_items, output_items)
