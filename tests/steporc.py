"""The light oracle's step with a count budget (TEST INFRASTRUCTURE: the checker, never the product): resumeorc.LightOracle
with the queue's highest priority (orc_light_queue_peek of oracle_light/liblightorc.so) and update_light_from_queue
(space/light/updater.rs:180-290) reporting LightUpdatesInfo (updater.rs:970-984)."""
import ctypes as C

import resumeorc

_ready = False


def lib():
    global _ready
    L = resumeorc.lib()
    if not _ready:
        L.orc_light_queue_peek.restype = C.c_int
        L.orc_light_queue_peek.argtypes = [C.c_void_p]
        _ready = True
    return L


class LightOracle(resumeorc.LightOracle):
    """resumeorc.LightOracle with the queue's highest priority and a budgeted step."""

    def queue_peek(self) -> int:
        """The highest queued priority; 0 (Priority::MIN) when the queue is empty."""
        return int(lib().orc_light_queue_peek(self.handle))

    def step(self, max_updates) -> dict:
        """update_light_from_queue with a budget of `max_updates` cube updates: pop the highest priority (lowest index
        within it) and apply it, one cube at a time, until the budget is spent or nothing above priority 1 is queued.
        The oracle's evaluate(0) is that loop; it leaves priority-1 entries, which the scenes of these tests never hold."""
        n, md = self.evaluate(0, max_updates)
        return {"update_count": n, "max_update_difference": md, "queue_count": self.queue_len(),
                "max_queue_priority": self.queue_peek()}
