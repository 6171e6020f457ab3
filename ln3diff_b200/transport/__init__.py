"""Mirror of the reference `transport` package (SiT flow matching), sampling side:
create_transport (transport/__init__.py:3-72), Transport.get_drift / get_score / check_interval
(transport/transport.py:85-112,193-245), Sampler.sample_ode (:374-421) and Sampler.sample_sde (:260-372), ode and sde
(integrators.py:9-120).  The fixed-grid solvers (euler, midpoint, heun, rk4) are implemented here; the adaptive
dopri5, bosh3, fehlberg2 and adaptive_heun delegate to torchdiffeq when it is installed (it is an un-vendored
third-party dependency of the reference, pinned 0.2.3) and otherwise run the restatement in rk.py."""
from .transport import (ModelType, PathType, Sampler, SNRType, Transport, WeightType, create_transport,  # noqa
                        sde_plan)
