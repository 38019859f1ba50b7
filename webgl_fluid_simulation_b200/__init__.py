"""H100-native (sm_90a) stable-fluids hot path behind the step()/splat()/config surface of
PavelDoGreat/WebGL-Fluid-Simulation.  See DESIGN.md; C ABI in include/fluid.h.

(The directory is `webgl_fluid_simulation_b200`: a hyphenated name cannot be imported in Python.)
"""
from ._lib import DISPLAY_BLOOM, DISPLAY_SHADING, DISPLAY_SUNRAYS, FIELD, PARAM, FLAG_HALF_POSTFX, FLAG_HALF_STORAGE, FLAG_LINEAR_ADVECTION, FLAG_NAIVE_JACOBI, FLAG_NEAREST_FILTERING, FLAG_NO_GRAPH, FLAG_TILED_PASSES, FLAG_UNFUSED, FluidError, build, lib  # noqa: F401
from .sim import FluidBatch, FluidSimulation, Pointer, capture_inputs, default_config, display_keywords, getResolution, HSVtoRGB, postfx_inputs, wrap, write_png  # noqa: F401
