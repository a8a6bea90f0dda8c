"""The light oracle with its update queue across save and load (TEST INFRASTRUCTURE: the checker, never the product):
physicsorc.LightOracle with the load rule of Space::new_from_builder, light_needs_update_in_region and a view of the
queue, orc_light_queue_uninitialized / orc_light_queue_region / orc_light_get_queue of oracle_light/liblightorc.so."""
import ctypes as C

import numpy as np

import physicsorc
from aicb200 import abi

_ready = False


def lib():
    global _ready
    L = physicsorc.lib()
    if not _ready:
        L.orc_light_queue_uninitialized.restype = C.c_size_t
        L.orc_light_queue_uninitialized.argtypes = [C.c_void_p]
        L.orc_light_queue_region.restype = C.c_int
        L.orc_light_queue_region.argtypes = [C.c_void_p, C.POINTER(abi.Aab), C.c_uint8]
        L.orc_light_get_queue.argtypes = [C.c_void_p, C.c_void_p]
        _ready = True
    return L


class LightOracle(physicsorc.LightOracle):
    """physicsorc.LightOracle whose queue can be resumed from a saved Space and read."""

    def queue_uninitialized(self) -> int:
        """Space::new_from_builder's load rule: every Uninitialized cube at Priority::UNINIT; returns their number."""
        return int(lib().orc_light_queue_uninitialized(self.handle))

    def queue_region(self, lower, size, priority):
        """light_needs_update_in_region; priority 0 raises ValueError and changes nothing."""
        region = abi.Aab()
        region.lower[:] = [int(v) for v in lower]
        region.size[:] = [int(v) for v in size]
        if lib().orc_light_queue_region(self.handle, C.byref(region), priority) != 0:
            raise ValueError("priority 0 never enters the queue")

    def queue(self) -> np.ndarray:
        """Each cube's queued priority (0 = not queued), uint8 shaped like the volume."""
        out = np.zeros(self.shape, dtype=np.uint8)
        lib().orc_light_get_queue(self.handle, out.ctypes.data)
        return out
