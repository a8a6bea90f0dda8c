"""An independent restatement of step_eye_position (all-is-cubes/src/character/eye.rs:90-121) and of the eye's view
transform (eye.rs:187-203) in numpy float64, operation by operation as euclid's vector operators evaluate them: every
array operation here is one correctly rounded IEEE operation per element, with nothing contracted."""
import math

import numpy as np

from aicb200 import abi


def step(eyes, bodies, dt):
    """One stepped tick of step_eye_position for eye i against body i, then previous_body_velocity = the body's
    velocity (what the next tick's record_previous_velocity reads).  eyes: abi.EYE_DTYPE, bodies: abi.BODY_DTYPE;
    returns new eyes."""
    with np.errstate(all="ignore"):   # huge displacements overflow to inf and NaN, as in the reference
        return _step(eyes, bodies, dt)


def _step(eyes, bodies, dt):
    e = np.array(eyes, dtype=abi.EYE_DTYPE, copy=True)
    v = np.asarray(bodies, dtype=abi.BODY_DTYPE)["velocity"].astype(np.float64)
    k21 = math.pow(1e21, dt)   # 1e21_f64.powf(dt)
    k9 = math.pow(1e-9, dt)    # 1e-9_f64.powf(dt)
    p = e["displacement_pos"].copy()
    vel = e["displacement_vel"].copy()
    # body_delta_v_this_frame = body.velocity() - previous_body_velocity; displacement_vel -= delta * 0.04
    vel = vel - (v - e["previous_body_velocity"]) * 0.04
    # displacement_vel -= displacement_pos * (displacement_pos.length() + 1.0) * 1e21^dt
    length = np.sqrt(p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2])
    vel = vel - (p * (length + 1.0)[:, None]) * k21
    # displacement_vel *= 1e-9^dt
    vel = vel * k9
    # displacement_pos += displacement_vel * dt
    p = p + vel * dt
    e["displacement_pos"] = p
    e["displacement_vel"] = vel
    e["previous_body_velocity"] = v
    return e


def eye_translation(eyes, bodies):
    """compute_view_transform's translation: body.position() + displacement_pos, float64 [n, 3]."""
    return (np.asarray(bodies, dtype=abi.BODY_DTYPE)["position"]
            + np.asarray(eyes, dtype=abi.EYE_DTYPE)["displacement_pos"])


def same_bytes(a, b) -> bool:
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.nbytes == b.nbytes and a.tobytes() == b.tobytes()
