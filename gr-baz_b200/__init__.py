"""gr-baz_b200: H100-native (sm_90a) drop-in for gr-baz's MUSIC direction-of-arrival block.

Only the hot path of /root/reference/lib/baz_music_doa.cc (work()) and its Python helper
(/root/reference/python/music_doa_helper.py) is rebuilt here; see DESIGN.md.
The directory name carries a hyphen, so it is imported through the ``gr_baz_b200`` alias
package at the repo root.
"""

from .music_doa_azel import music_doa_azel  # noqa: E402,F401  (azimuth + elevation, include/music_b200.h)
from .music_doa_channels import music_doa_channels  # noqa: E402,F401  (frequency-channelised, include/music_b200.h)
from .music_doa_coarray import music_doa_coarray  # noqa: E402,F401  (sparse linear arrays, include/music_b200.h)
