"""Hand-written sm_90a operators (ctypes bindings over csrc/)."""
