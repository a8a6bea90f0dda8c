"""The light oracle with a changing physics (TEST INFRASTRUCTURE: the checker, never the product): lightorc.LightOracle
with SpaceChange::Physics on the light side, orc_light_set_physics of oracle_light/liblightorc.so."""
import ctypes as C

import lightorc
from aicb200 import _sky, abi

_ready = False


def lib():
    global _ready
    L = lightorc.lib()
    if not _ready:
        L.orc_light_set_physics.argtypes = [C.c_void_p, C.POINTER(abi.Sky), C.c_uint8]
        _ready = True
    return L


class LightOracle(lightorc.LightOracle):
    """lightorc.LightOracle whose sky and LightPhysics change after creation."""

    def set_physics(self, sky_colors, light_max_distance):
        """maybe_reinitialize_for_physics_change: the new BlockSky; a new LightPhysics reinitialises (fast_evaluate)."""
        lib().orc_light_set_physics(self.handle, C.byref(_sky(sky_colors)), light_max_distance)
