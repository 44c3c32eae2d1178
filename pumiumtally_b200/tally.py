"""Python host-side mirror of ``pumitally::PumiTally`` over the C ABI.

Same method names and argument meaning as the reference class
(reference: src/pumitally/PumiTally.h:50-103) so parity tests read like the
reference's own test (test/test_pumi_tally_impl_methods.cpp).  Every call goes
through ``libpumitally.so`` (include/pumitally_c.h); there is no Python or CPU
implementation of the path behind this class -- if the CUDA library is missing
or no GPU is present, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
# PUMITALLY_LIB selects another build of the same library (tests of the measured alternative kernels
# use lib/libpumitally_exp.so); the default is the product library.
LIB_PATH = os.environ.get("PUMITALLY_LIB") or os.path.join(_PKG, "lib", "libpumitally.so")
_lib = None

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)
_bp = C.POINTER(C.c_int8)
_u8p = C.POINTER(C.c_uint8)


class Stats(C.Structure):
    _fields_ = [
        ("segments", C.c_uint64), ("tracks", C.c_uint64), ("relocations", C.c_uint64),
        ("lost", C.c_uint64), ("moves", C.c_uint64), ("kernel_ms", C.c_double),
        ("h2d_bytes", C.c_double), ("plane_fallbacks", C.c_uint64),
    ]


# name -> (restype, argtypes); also the list tests check against include/pumitally_c.h
C_API = {
    "pumitally_create": (C.c_void_p, [C.c_char_p, C.c_int32, C.POINTER(C.c_int), C.c_void_p]),
    "pumitally_copy_initial_position": (C.c_int, [C.c_void_p, _dp, C.c_int32]),
    "pumitally_move_to_next_location": (C.c_int, [C.c_void_p, _dp, _dp, _bp, _dp, C.c_int32]),
    "pumitally_move_to_next_location_binned": (C.c_int, [C.c_void_p, _dp, _dp, _bp, _dp, _ip, C.c_int32]),
    "pumitally_move_to_next_location_device_binned": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "pumitally_set_score_bins": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_get_score_bins": (C.c_int32, [C.c_void_p]),
    "pumitally_set_scores": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_get_scores": (C.c_int32, [C.c_void_p]),
    "pumitally_move_to_next_location_scored": (C.c_int, [C.c_void_p, _dp, _dp, _bp, _dp, _dp, _ip, C.c_int32]),
    "pumitally_move_to_next_location_device_scored": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                  C.c_void_p]),
    "pumitally_set_time_bins": (C.c_int, [C.c_void_p, _dp, C.c_int32]),
    "pumitally_get_time_bins": (C.c_int32, [C.c_void_p]),
    "pumitally_move_to_next_location_timed": (C.c_int, [C.c_void_p, _dp, _dp, _bp, _dp, _dp, _dp, _dp, _ip, C.c_int32]),
    "pumitally_move_to_next_location_device_timed": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_int32, C.c_void_p]),
    "pumitally_set_moments": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_get_moments": (C.c_int32, [C.c_void_p]),
    "pumitally_get_flux_moments": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pumitally_get_flux_gradient": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pumitally_locate_points": (C.c_int, [C.c_void_p, _dp, C.c_int64, _ip]),
    "pumitally_locate_points_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "pumitally_evaluate_points": (C.c_int, [C.c_void_p, _dp, C.c_int64, _dp, C.c_int64, _ip]),
    "pumitally_set_collision_estimator": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_get_collision_estimator": (C.c_int32, [C.c_void_p]),
    "pumitally_set_face_currents": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_get_face_currents": (C.c_int32, [C.c_void_p]),
    "pumitally_get_face_current_results": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _dp, C.c_int64]),
    "pumitally_get_leakage": (C.c_int, [C.c_void_p, C.c_int32, _dp, C.c_int64]),
    "pumitally_set_current_cosine_bins": (C.c_int, [C.c_void_p, _dp, C.c_int32]),
    "pumitally_get_current_cosine_bins": (C.c_int32, [C.c_void_p]),
    "pumitally_tally_collisions": (C.c_int, [C.c_void_p, _dp, C.c_int64, _dp, _dp, _ip, _dp]),
    "pumitally_tally_collisions_device": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pumitally_tally_collisions_at_particles": (C.c_int, [C.c_void_p, _bp, _dp, _dp, _ip, _dp, C.c_int32]),
    "pumitally_tally_collisions_at_particles_device": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "pumitally_get_collision_results": (C.c_int, [C.c_void_p, C.c_int32, _dp, C.c_int64]),
    "pumitally_set_point_detectors": (C.c_int, [C.c_void_p, _dp, C.c_int32, _dp]),
    "pumitally_get_point_detectors": (C.c_int32, [C.c_void_p]),
    "pumitally_set_detector_cross_sections": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pumitally_set_detector_void": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_get_detector_void": (C.c_int32, [C.c_void_p]),
    "pumitally_tally_detectors": (C.c_int, [C.c_void_p, _dp, C.c_int64, _dp, _dp, _dp, _ip, _dp, _dp]),
    "pumitally_tally_detectors_device": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_void_p, C.c_void_p]),
    "pumitally_tally_detectors_at_particles": (C.c_int, [C.c_void_p, _bp, _dp, _dp, _dp, _ip, _dp, _dp, C.c_int32]),
    "pumitally_tally_detectors_at_particles_device": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_int32, C.c_void_p]),
    "pumitally_get_detector_results": (C.c_int, [C.c_void_p, C.c_int32, _dp, C.c_int64]),
    "pumitally_set_batch_statistics": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_end_batch": (C.c_int, [C.c_void_p]),
    "pumitally_get_batch_results": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _dp, C.c_int64]),
    "pumitally_get_batch_max_rel_err": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _dp, C.POINTER(C.c_int64)]),
    "pumitally_set_regions": (C.c_int, [C.c_void_p, _ip, C.c_int64, C.c_int32]),
    "pumitally_get_regions": (C.c_int32, [C.c_void_p]),
    "pumitally_get_region_volumes": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pumitally_get_region_results": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _dp, C.c_int64]),
    "pumitally_get_region_batch_results": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _dp, C.c_int64]),
    "pumitally_set_region_currents": (C.c_int, [C.c_void_p, C.c_int32]),
    "pumitally_get_region_currents": (C.c_int32, [C.c_void_p]),
    "pumitally_get_region_current_pair_count": (C.c_int64, [C.c_void_p]),
    "pumitally_get_region_current_pairs": (C.c_int, [C.c_void_p, _ip, _ip, C.c_int64]),
    "pumitally_get_region_current_areas": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pumitally_get_region_current_results": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _dp, C.c_int64]),
    "pumitally_save_checkpoint": (C.c_int, [C.c_void_p, C.c_char_p]),
    "pumitally_load_checkpoint": (C.c_int, [C.c_void_p, C.c_char_p]),
    "pumitally_merge_checkpoint": (C.c_int, [C.c_void_p, C.c_char_p]),
    "pumitally_set_weight_windows": (C.c_int, [C.c_void_p, _dp, _dp, C.c_int64, C.c_int32]),
    "pumitally_get_weight_window_groups": (C.c_int32, [C.c_void_p]),
    "pumitally_get_weight_windows": (C.c_int, [C.c_void_p, _dp, _dp, C.c_int64]),
    "pumitally_generate_weight_windows": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                                    C.c_double]),
    "pumitally_get_weight_windows_at_particles": (C.c_int, [C.c_void_p, _ip, _dp, _dp, C.c_int32]),
    "pumitally_get_weight_windows_at_particles_device": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "pumitally_get_weight_windows_at_points": (C.c_int, [C.c_void_p, _dp, C.c_int64, _ip, _dp, _dp]),
    "pumitally_get_weight_windows_at_points_device": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pumitally_set_source": (C.c_int, [C.c_void_p, _dp, _dp, C.c_int64, C.c_int32, C.c_int32]),
    "pumitally_get_source_groups": (C.c_int32, [C.c_void_p]),
    "pumitally_get_source_strength": (C.c_int, [C.c_void_p, _dp]),
    "pumitally_sample_source": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int64, C.c_int64, _dp, _ip, _ip, _dp, C.c_int32]),
    "pumitally_sample_source_device": (
        C.c_int, [C.c_void_p, C.c_uint64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                  C.c_int32, C.c_void_p]),
    "pumitally_write_tally_results": (C.c_int, [C.c_void_p]),
    "pumitally_destroy": (None, [C.c_void_p]),
    "pumitally_create_from_arrays": (C.c_void_p, [_dp, C.c_int64, _ip, C.c_int64, C.c_int32, C.c_int32]),
    "pumitally_num_elements": (C.c_int64, [C.c_void_p]),
    "pumitally_num_particles": (C.c_int32, [C.c_void_p]),
    "pumitally_get_flux": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pumitally_get_normalized_flux": (C.c_int, [C.c_void_p, _dp, _dp, C.c_int64]),
    "pumitally_get_element_ids": (C.c_int, [C.c_void_p, _ip, C.c_int64]),
    "pumitally_get_positions": (C.c_int, [C.c_void_p, _dp, C.c_int64]),
    "pumitally_get_adjacency": (C.c_int, [C.c_void_p, _ip, C.c_int64]),
    "pumitally_reset_tally": (C.c_int, [C.c_void_p]),
    "pumitally_set_source_normalization": (C.c_int, [C.c_void_p, C.c_int32, C.c_double]),
    "pumitally_get_source_normalization": (C.c_double, [C.c_void_p]),
    "pumitally_get_stats": (C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    "pumitally_set_output_name": (C.c_int, [C.c_void_p, C.c_char_p]),
    "pumitally_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    "pumitally_get_option": (C.c_int64, [C.c_void_p, C.c_char_p]),
    "pumitally_copy_initial_position_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "pumitally_move_to_next_location_device": (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "pumitally_set_state_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "pumitally_get_state_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "pumitally_get_flux_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "pumitally_flux_device_ptr": (C.c_void_p, [C.c_void_p]),
    "pumitally_synchronize": (C.c_int, [C.c_void_p]),
    "pumitally_nccl_unique_id": (C.c_int, [_u8p]),
    "pumitally_comm_init": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _u8p]),
    "pumitally_allreduce_tally": (C.c_int, [C.c_void_p]),
    "pumitally_reduce_tally_to_owners": (C.c_int, [C.c_void_p]),
    "pumitally_exchange_tally": (C.c_int, [C.c_void_p]),
    "pumitally_debug_order": (C.c_int64, [C.c_void_p, _ip, C.c_int64]),
    "pumitally_debug_stage": (C.c_int64, [_dp, _dp, _bp, _dp, _dp, _dp, _bp, C.c_int64, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_int64]),
    "pumitally_version": (C.c_char_p, []),
}


def load_library():
    """dlopen libpumitally.so and declare the C ABI. Raises if it was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`."
                " There is no CPU implementation of the tally path in this package.")
        L = C.CDLL(LIB_PATH)
        for name, (rt, at) in C_API.items():
            fn = getattr(L, name)
            fn.restype = rt
            fn.argtypes = at
        _lib = L
    return _lib


def _host_f64(a, what):
    a = np.asarray(a)
    if a.dtype != np.float64 or not a.flags.c_contiguous:
        a = np.ascontiguousarray(a, dtype=np.float64)
    return a.reshape(-1)


class PumiTally:
    """Track-length tally engine on one H100.

    ``PumiTally(mesh_filename, num_particles)`` follows the reference constructor;
    ``PumiTally.from_arrays(coords, tet2vert, num_particles)`` takes the mesh in memory.
    """

    def __init__(self, mesh_filename: str, num_particles: int, argv=None, _handle=None):
        self._L = load_library()
        self.num_particles = int(num_particles)
        if _handle is None:
            argc = C.c_int(0)
            _handle = self._L.pumitally_create(str(mesh_filename).encode(), self.num_particles,
                                               C.byref(argc), None)
        if not _handle:
            raise RuntimeError("pumitally engine construction failed (mesh unreadable or no CUDA device)")
        self._h = C.c_void_p(_handle)
        self.num_elements = int(self._L.pumitally_num_elements(self._h))

    @classmethod
    def from_spec(cls, mesh_filename: str, num_particles: int, device: int = -1):
        """Reference constructor with the CUDA device passed the way the reference passes
        runtime options: through argv (``--pumitally-device=<id>``)."""
        L = load_library()
        args = [b"pumitally"] + ([f"--pumitally-device={device}".encode()] if device >= 0 else [])
        argv = (C.c_char_p * (len(args) + 1))(*args, None)
        argc = C.c_int(len(args))
        argv_p = C.cast(argv, C.POINTER(C.c_char_p))
        h = L.pumitally_create(str(mesh_filename).encode(), int(num_particles), C.byref(argc), C.byref(argv_p))
        if not h:
            raise RuntimeError("pumitally engine construction failed (mesh unreadable or no CUDA device)")
        return cls("", num_particles, _handle=h)

    @classmethod
    def from_arrays(cls, coords, tet2vert, num_particles: int, device: int = -1):
        L = load_library()
        coords = np.ascontiguousarray(coords, dtype=np.float64)
        t2v = np.ascontiguousarray(tet2vert, dtype=np.int32)
        h = L.pumitally_create_from_arrays(coords.ctypes.data_as(_dp), coords.shape[0],
                                           t2v.ctypes.data_as(_ip), t2v.shape[0],
                                           int(num_particles), int(device))
        if not h:
            raise RuntimeError("pumitally engine construction failed (bad mesh or no CUDA device)")
        return cls("", num_particles, _handle=h)

    def close(self):
        if getattr(self, "_h", None):
            self._L.pumitally_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- reference interface -------------------------------------------------
    def CopyInitialPosition(self, init_particle_positions, size=None):
        xyz = _host_f64(init_particle_positions, "init_particle_positions")
        size = xyz.size if size is None else int(size)
        if self._L.pumitally_copy_initial_position(self._h, xyz.ctypes.data_as(_dp), size):
            raise RuntimeError("CopyInitialPosition failed")

    def MoveToNextLocation(self, particle_origin, particle_destinations, flying, weights, size=None):
        o = _host_f64(particle_origin, "particle_origin")
        d = _host_f64(particle_destinations, "particle_destinations")
        w = _host_f64(weights, "weights")
        if not (isinstance(flying, np.ndarray) and flying.dtype == np.int8 and flying.flags.c_contiguous):
            raise TypeError("flying must be a contiguous int8 numpy array (the engine zeroes it)")
        size = o.size if size is None else int(size)
        if self._L.pumitally_move_to_next_location(self._h, o.ctypes.data_as(_dp), d.ctypes.data_as(_dp),
                                                   flying.ctypes.data_as(_bp), w.ctypes.data_as(_dp), size):
            raise RuntimeError("MoveToNextLocation failed")

    # ---- score filter ----------------------------------------------------------
    def set_score_bins(self, nbins: int):
        """nbins flux arrays (resets the tally); binned moves score particle i into array bins[i]."""
        if self._L.pumitally_set_score_bins(self._h, int(nbins)):
            raise ValueError(f"set_score_bins({nbins}) failed")

    @property
    def score_bins(self) -> int:
        return int(self._L.pumitally_get_score_bins(self._h))

    def MoveToNextLocationBinned(self, particle_origin, particle_destinations, flying, weights, bins, size=None):
        o = _host_f64(particle_origin, "particle_origin")
        d = _host_f64(particle_destinations, "particle_destinations")
        w = _host_f64(weights, "weights")
        if not (isinstance(flying, np.ndarray) and flying.dtype == np.int8 and flying.flags.c_contiguous):
            raise TypeError("flying must be a contiguous int8 numpy array (the engine zeroes it)")
        if not (isinstance(bins, np.ndarray) and bins.dtype == np.int32 and bins.flags.c_contiguous and bins.size == w.size):
            raise TypeError("bins must be a contiguous int32 numpy array, one entry per particle")
        size = o.size if size is None else int(size)
        if self._L.pumitally_move_to_next_location_binned(self._h, o.ctypes.data_as(_dp), d.ctypes.data_as(_dp),
                                                          flying.ctypes.data_as(_bp), w.ctypes.data_as(_dp),
                                                          bins.ctypes.data_as(_ip), size):
            raise RuntimeError("MoveToNextLocationBinned failed")

    def move_device_binned(self, d_origin, d_dest, d_flying, d_weights, d_bins, stream=None):
        if self._L.pumitally_move_to_next_location_device_binned(self._h, d_origin, d_dest, d_flying, d_weights, d_bins,
                                                                 3 * self.num_particles, stream):
            raise RuntimeError("MoveToNextLocationBinned(device) failed")

    @property
    def flux_bins(self):
        """Raw flux of every score bin: array [nbins, num_elements]."""
        out = np.empty((self.score_bins, self.num_elements))
        if self._L.pumitally_get_flux(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_flux failed")
        return out

    def normalized_flux_bins(self):
        f, v = np.empty((self.score_bins, self.num_elements)), np.empty(self.num_elements)
        if self._L.pumitally_get_normalized_flux(self._h, f.ctypes.data_as(_dp), v.ctypes.data_as(_dp), f.size):
            raise RuntimeError("get_normalized_flux failed")
        return f, v

    # ---- scores ------------------------------------------------------------------
    def set_scores(self, nscores: int):
        """nscores responses per particle, tallied in one walk (resets the tally); 1 <= nscores <= 8."""
        if self._L.pumitally_set_scores(self._h, int(nscores)):
            raise ValueError(f"set_scores({nscores}) failed")

    @property
    def scores(self) -> int:
        return int(self._L.pumitally_get_scores(self._h))

    def MoveToNextLocationScored(self, particle_origin, particle_destinations, flying, weights, responses, bins=None,
                                 size=None):
        """Score k of every segment gets length * weights[i] * responses[i, k]; responses: [num_particles, nscores]."""
        o = _host_f64(particle_origin, "particle_origin")
        d = _host_f64(particle_destinations, "particle_destinations")
        w = _host_f64(weights, "weights")
        r = _host_f64(responses, "responses")
        if not (isinstance(flying, np.ndarray) and flying.dtype == np.int8 and flying.flags.c_contiguous):
            raise TypeError("flying must be a contiguous int8 numpy array (the engine zeroes it)")
        if r.size != w.size * self.scores:
            raise TypeError(f"responses must hold num_particles * {self.scores} values")
        bp = None
        if bins is not None:
            if not (isinstance(bins, np.ndarray) and bins.dtype == np.int32 and bins.flags.c_contiguous and bins.size == w.size):
                raise TypeError("bins must be a contiguous int32 numpy array, one entry per particle")
            bp = bins.ctypes.data_as(_ip)
        size = o.size if size is None else int(size)
        if self._L.pumitally_move_to_next_location_scored(self._h, o.ctypes.data_as(_dp), d.ctypes.data_as(_dp),
                                                          flying.ctypes.data_as(_bp), w.ctypes.data_as(_dp),
                                                          r.ctypes.data_as(_dp), bp, size):
            raise RuntimeError("MoveToNextLocationScored failed")

    def move_device_scored(self, d_origin, d_dest, d_flying, d_weights, d_responses, d_bins=None, stream=None):
        """Scored move on device addresses (responses particle-major); enqueues on ``stream`` and returns."""
        if self._L.pumitally_move_to_next_location_device_scored(self._h, d_origin, d_dest, d_flying, d_weights,
                                                                 d_responses, d_bins, 3 * self.num_particles, stream):
            raise RuntimeError("MoveToNextLocationScored(device) failed")

    @property
    def flux_scores(self):
        """Raw flux of every score bin and score: array [nbins, nscores, num_elements]."""
        out = np.empty((self.score_bins, self.scores, self.num_elements))
        if self._L.pumitally_get_flux(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_flux failed")
        return out

    def normalized_flux_scores(self):
        f, v = np.empty((self.score_bins, self.scores, self.num_elements)), np.empty(self.num_elements)
        if self._L.pumitally_get_normalized_flux(self._h, f.ctypes.data_as(_dp), v.ctypes.data_as(_dp), f.size):
            raise RuntimeError("get_normalized_flux failed")
        return f, v

    # ---- time filter -------------------------------------------------------------
    def set_time_bins(self, edges):
        """Time bins [edges[j], edges[j+1]) (finite, strictly increasing, 2..1025 edges; resets the tally).
        ``None`` removes the filter."""
        if edges is None:
            rc = self._L.pumitally_set_time_bins(self._h, None, 0)
        else:
            e = np.ascontiguousarray(edges, dtype=np.float64).reshape(-1)
            rc = self._L.pumitally_set_time_bins(self._h, e.ctypes.data_as(_dp), int(e.size))
        if rc:
            raise ValueError("set_time_bins failed")

    @property
    def time_bins(self) -> int:
        """Number of time bins, 0 without a time filter."""
        return int(self._L.pumitally_get_time_bins(self._h))

    def MoveToNextLocationTimed(self, particle_origin, particle_destinations, flying, weights, times, speeds,
                                responses=None, bins=None, size=None):
        """Scored move whose segments are split between the time bins they span: times[i] is particle i's time at
        its origin, speeds[i] its speed (mesh length units per time unit).  responses may be None with one score."""
        o = _host_f64(particle_origin, "particle_origin")
        d = _host_f64(particle_destinations, "particle_destinations")
        w = _host_f64(weights, "weights")
        t = _host_f64(times, "times")
        v = _host_f64(speeds, "speeds")
        if not (isinstance(flying, np.ndarray) and flying.dtype == np.int8 and flying.flags.c_contiguous):
            raise TypeError("flying must be a contiguous int8 numpy array (the engine zeroes it)")
        if t.size != w.size or v.size != w.size:
            raise TypeError("times and speeds must hold one value per particle")
        rp = None
        if responses is not None:
            r = _host_f64(responses, "responses")
            if r.size != w.size * self.scores:
                raise TypeError(f"responses must hold num_particles * {self.scores} values")
            rp = r.ctypes.data_as(_dp)
        bp = None
        if bins is not None:
            if not (isinstance(bins, np.ndarray) and bins.dtype == np.int32 and bins.flags.c_contiguous and bins.size == w.size):
                raise TypeError("bins must be a contiguous int32 numpy array, one entry per particle")
            bp = bins.ctypes.data_as(_ip)
        size = o.size if size is None else int(size)
        if self._L.pumitally_move_to_next_location_timed(self._h, o.ctypes.data_as(_dp), d.ctypes.data_as(_dp),
                                                         flying.ctypes.data_as(_bp), w.ctypes.data_as(_dp),
                                                         t.ctypes.data_as(_dp), v.ctypes.data_as(_dp), rp, bp, size):
            raise RuntimeError("MoveToNextLocationTimed failed")

    def move_device_timed(self, d_origin, d_dest, d_flying, d_weights, d_times, d_speeds, d_responses=None, d_bins=None,
                          stream=None):
        """Timed move on device addresses; enqueues on ``stream`` and returns."""
        if self._L.pumitally_move_to_next_location_device_timed(self._h, d_origin, d_dest, d_flying, d_weights, d_times,
                                                                d_speeds, d_responses, d_bins, 3 * self.num_particles,
                                                                stream):
            raise RuntimeError("MoveToNextLocationTimed(device) failed")

    @property
    def flux_time(self):
        """Raw flux of every time bin, score bin and score: array [ntime, nbins, nscores, num_elements]."""
        out = np.empty((max(self.time_bins, 1), self.score_bins, self.scores, self.num_elements))
        if self._L.pumitally_get_flux(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_flux failed")
        return out

    def normalized_flux_time(self):
        f = np.empty((max(self.time_bins, 1), self.score_bins, self.scores, self.num_elements))
        v = np.empty(self.num_elements)
        if self._L.pumitally_get_normalized_flux(self._h, f.ctypes.data_as(_dp), v.ctypes.data_as(_dp), f.size):
            raise RuntimeError("get_normalized_flux failed")
        return f, v

    # ---- linear flux moments -------------------------------------------------------
    def set_moments(self, order: int):
        """1: every move also tallies the first spatial moment of each score in each element; 0: no moments (the
        default).  Resets the tally."""
        if self._L.pumitally_set_moments(self._h, int(order)):
            raise ValueError("set_moments failed")

    @property
    def moments(self) -> int:
        """Moment order, 0 without moments."""
        return int(self._L.pumitally_get_moments(self._h))

    def _moment_array(self, fn, what):
        out = np.empty((max(self.time_bins, 1), self.score_bins, self.scores, self.num_elements, 3))
        if fn(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError(f"{what} failed")
        return out

    def flux_moments(self):
        """Raw first moments about each element's centroid: array [ntime, nbins, nscores, num_elements, 3]."""
        return self._moment_array(self._L.pumitally_get_flux_moments, "get_flux_moments")

    def flux_gradient(self):
        """Normalised flux gradient of each element's linear flux, shaped as flux_moments()."""
        return self._moment_array(self._L.pumitally_get_flux_gradient, "get_flux_gradient")

    # ---- point queries -------------------------------------------------------------
    @staticmethod
    def _points(points):
        p = _host_f64(points, "points")
        if p.size % 3:
            raise TypeError("points must hold x, y, z per point")
        return p, p.size // 3

    def locate(self, points):
        """Element (caller's numbering) containing each point of ``points`` [npts, 3]; -1 outside the mesh."""
        p, npts = self._points(points)
        out = np.empty(npts, dtype=np.int32)
        if self._L.pumitally_locate_points(self._h, p.ctypes.data_as(_dp), npts, out.ctypes.data_as(_ip)):
            raise RuntimeError("locate_points failed")
        return out

    def locate_device(self, points, stream=None):
        """locate() on a contiguous float64 CUDA tensor [npts, 3]: returns an int32 CUDA tensor, enqueued on ``stream``
        (default: the current torch stream)."""
        import torch

        if not (points.is_cuda and points.dtype == torch.float64 and points.is_contiguous() and points.numel() % 3 == 0):
            raise TypeError("points must be a contiguous float64 CUDA tensor of shape [npts, 3]")
        npts = points.numel() // 3
        out = torch.empty(npts, dtype=torch.int32, device=points.device)
        if stream is None:
            stream = torch.cuda.current_stream(points.device).cuda_stream
        if self._L.pumitally_locate_points_device(self._h, points.data_ptr(), npts, out.data_ptr(), stream):
            raise RuntimeError("locate_points_device failed")
        return out

    def evaluate(self, points, first_only=False):
        """Normalised results at the points: (values [ntime, nbins, nscores, npts] -- the linear reconstruction with
        moments, NaN outside the mesh -- and the elements as locate() gives them).  first_only: values [npts] of time
        bin 0, bin 0, score 0."""
        p, npts = self._points(points)
        shape = (npts,) if first_only else (max(self.time_bins, 1), self.score_bins, self.scores, npts)
        out = np.empty(shape)
        elem = np.empty(npts, dtype=np.int32)
        if self._L.pumitally_evaluate_points(self._h, p.ctypes.data_as(_dp), npts, out.ctypes.data_as(_dp), out.size,
                                             elem.ctypes.data_as(_ip)):
            raise RuntimeError("evaluate_points failed")
        return out, elem

    # ---- face currents ---------------------------------------------------------------
    def set_face_currents(self, on: bool):
        """True: every move also tallies the weight crossing each element face, per score bin and time bin, and the
        leakage through the hull; False stops it (the default).  Resets the tally and discards the folded batches."""
        if self._L.pumitally_set_face_currents(self._h, int(on)):
            raise ValueError("set_face_currents failed")

    @property
    def face_currents(self) -> bool:
        return bool(self._L.pumitally_get_face_currents(self._h))

    def set_current_cosine_bins(self, edges):
        """Cosine bins of the face currents: edges mu_0 < ... < mu_C in [0, 1] (2..65 of them; resets the tally and
        discards the folded batches).  Every crossing also goes to the bin of the cosine between its flight and the
        face normal that points the way it travels; face_current_results, leakage and region_current_results gain an
        axis of C cosine bins after the score-bin axis.  ``None`` removes them."""
        if edges is None:
            rc = self._L.pumitally_set_current_cosine_bins(self._h, None, 0)
        else:
            e = np.ascontiguousarray(edges, dtype=np.float64).reshape(-1)
            rc = self._L.pumitally_set_current_cosine_bins(self._h, e.ctypes.data_as(_dp), int(e.size))
        if rc:
            raise ValueError("set_current_cosine_bins failed")

    @property
    def current_cosine_bins(self) -> int:
        """Number of cosine bins of the face currents, 0 without them."""
        return int(self._L.pumitally_get_current_cosine_bins(self._h))

    def _cosine_axis(self):
        C = self.current_cosine_bins
        return (C,) if C > 0 else ()

    def face_current_results(self, direction=0, kind=0):
        """Partial currents [ntime, nbins, (C,) num_elements, 4] in the caller's numbering, face f opposite local
        vertex f (the cosine axis only while cosine bins are set): direction 0 outgoing, 1 incoming; kind 0 the open
        tally / the per-source divisor, 1 batch mean, 2 standard error, 3 relative error."""
        out = np.empty((max(self.time_bins, 1), self.score_bins) + self._cosine_axis() + (self.num_elements, 4))
        if self._L.pumitally_get_face_current_results(self._h, int(direction), int(kind), out.ctypes.data_as(_dp),
                                                      out.size):
            raise RuntimeError("get_face_current_results failed")
        return out

    def leakage(self, kind=0):
        """The outgoing current summed over the hull faces, [ntime, nbins, (C)]; kinds as face_current_results."""
        out = np.empty((max(self.time_bins, 1), self.score_bins) + self._cosine_axis())
        if self._L.pumitally_get_leakage(self._h, int(kind), out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_leakage failed")
        return out

    # ---- collision estimator -------------------------------------------------------
    def set_collision_estimator(self, on: bool):
        """True: a collision tally with the track-length tally's configuration, in arrays of its own (resets the
        tally); False removes it."""
        if self._L.pumitally_set_collision_estimator(self._h, int(on)):
            raise ValueError("set_collision_estimator failed")

    @property
    def collision_estimator(self) -> bool:
        return bool(self._L.pumitally_get_collision_estimator(self._h))

    def _event_args(self, n, weights, responses, bins, times, pdf=None, speeds=None):
        """Host event arrays as contiguous numpy arrays (None stays None), checked against n events: (arrays, pointers
        to weights, responses, bins, times, pdf [n, point_detectors] and speeds)."""
        w = _host_f64(weights, "weights")
        if w.size != n:
            raise TypeError("weights must hold one value per event")
        r = t = b = p = v = None
        if responses is not None:
            r = _host_f64(responses, "responses")
            if r.size != n * self.scores:
                raise TypeError(f"responses must hold {self.scores} values per event")
        if times is not None:
            t = _host_f64(times, "times")
            if t.size != n:
                raise TypeError("times must hold one value per event")
        if bins is not None:
            b = np.ascontiguousarray(bins, dtype=np.int32).reshape(-1)
            if b.size != n:
                raise TypeError("bins must hold one value per event")
        if pdf is not None:
            p = _host_f64(pdf, "pdf")
            if p.size != n * self.point_detectors:
                raise TypeError(f"pdf must hold {self.point_detectors} values per event")
        if speeds is not None:
            v = _host_f64(speeds, "speeds")
            if v.size != n:
                raise TypeError("speeds must hold one value per event")
        ptr = lambda a, q: None if a is None else a.ctypes.data_as(q)  # noqa: E731
        return (w, r, b, t, p, v), (ptr(w, _dp), ptr(r, _dp), ptr(b, _ip), ptr(t, _dp), ptr(p, _dp), ptr(v, _dp))

    def tally_collisions(self, points, weights, responses=None, bins=None, times=None):
        """Collision events at ``points`` [n, 3], each located as locate() does: event i adds weights[i] *
        responses[i, k] to score k of its element, bin bins[i] and the time bin of times[i]."""
        p, n = self._points(points)
        _keep, (w, r, b, t, _, _) = self._event_args(n, weights, responses, bins, times)
        if self._L.pumitally_tally_collisions(self._h, p.ctypes.data_as(_dp), n, w, r, b, t):
            raise RuntimeError("tally_collisions failed")

    @staticmethod
    def _tensor_ptr(x, dtype, numel, what):
        if x is None:
            return None
        if not (x.is_cuda and x.dtype == dtype and x.is_contiguous() and x.numel() == numel):
            raise TypeError(f"{what} must be a contiguous {dtype} CUDA tensor of {numel} values")
        return x.data_ptr()

    def _device_event_args(self, n, weights, responses, bins, times, stream, device, pdf=None, speeds=None):
        """Device pointers of weights, responses, bins, times, pdf [n, point_detectors] and speeds, and the stream."""
        import torch

        args = (self._tensor_ptr(weights, torch.float64, n, "weights"),
                self._tensor_ptr(responses, torch.float64, n * self.scores, "responses"),
                self._tensor_ptr(bins, torch.int32, n, "bins"),
                self._tensor_ptr(times, torch.float64, n, "times"),
                self._tensor_ptr(pdf, torch.float64, n * self.point_detectors, "pdf"),
                self._tensor_ptr(speeds, torch.float64, n, "speeds"))
        if stream is None:
            stream = torch.cuda.current_stream(device).cuda_stream
        return args, stream

    def tally_collisions_device(self, points, weights, responses=None, bins=None, times=None, stream=None):
        """tally_collisions() on CUDA tensors (points float64 [n, 3], weights and times float64 [n], responses
        float64 [n, nscores], bins int32 [n]); enqueued on ``stream`` (default: the current torch stream)."""
        import torch

        if not (points.is_cuda and points.dtype == torch.float64 and points.is_contiguous() and points.numel() % 3 == 0):
            raise TypeError("points must be a contiguous float64 CUDA tensor of shape [n, 3]")
        n = points.numel() // 3
        (w, r, b, t, _, _), stream = self._device_event_args(n, weights, responses, bins, times, stream, points.device)
        if self._L.pumitally_tally_collisions_device(self._h, points.data_ptr(), n, w, r, b, t, stream):
            raise RuntimeError("tally_collisions_device failed")

    def tally_collisions_at_particles(self, collided, weights, responses=None, bins=None, times=None):
        """Collision events at the stored positions of the particles i with collided[i] != 0, in their elements."""
        c = np.ascontiguousarray(collided, dtype=np.int8).reshape(-1)
        _keep, (w, r, b, t, _, _) = self._event_args(c.size, weights, responses, bins, times)
        if self._L.pumitally_tally_collisions_at_particles(self._h, c.ctypes.data_as(_bp), w, r, b, t, c.size):
            raise RuntimeError("tally_collisions_at_particles failed")

    def tally_collisions_at_particles_device(self, collided, weights, responses=None, bins=None, times=None,
                                             stream=None):
        """tally_collisions_at_particles() on CUDA tensors (collided int8 [num_particles]); enqueued on ``stream``."""
        import torch

        n = self.num_particles
        c = self._tensor_ptr(collided, torch.int8, n, "collided")
        (w, r, b, t, _, _), stream = self._device_event_args(n, weights, responses, bins, times, stream,
                                                             collided.device)
        if self._L.pumitally_tally_collisions_at_particles_device(self._h, c, w, r, b, t, n, stream):
            raise RuntimeError("tally_collisions_at_particles_device failed")

    def collision_results(self, kind=0):
        """The collision tally: kind 0 raw, 1 normalised ([ntime, nbins, nscores, num_elements]), 2 first moments, 3
        gradient ([..., 3]) -- what flux_time, normalized_flux_time()[0], flux_moments() and flux_gradient() give for
        the track-length tally."""
        shape = (max(self.time_bins, 1), self.score_bins, self.scores, self.num_elements) + ((3,) if kind in (2, 3) else ())
        out = np.empty(shape)
        if self._L.pumitally_get_collision_results(self._h, int(kind), out.ctypes.data_as(_dp), out.size):
            raise RuntimeError(f"get_collision_results({kind}) failed")
        return out

    # ---- point detectors -----------------------------------------------------------
    def set_point_detectors(self, points, r0):
        """Next-event (point-detector) estimates at ``points`` [D, 3] (1 <= D <= 256, inside the mesh, or anywhere
        finite with the detector void on: set_detector_void) with exclusion
        radii ``r0`` [D] (finite, >= 0).  ``points`` None removes them.  Resets the tally and discards the folded
        batches."""
        if points is None:
            rc = self._L.pumitally_set_point_detectors(self._h, None, 0, None)
        else:
            p = _host_f64(points, "points")
            r = _host_f64(r0, "r0")
            if p.size % 3 or r.size != p.size // 3:
                raise TypeError("points must be [D, 3] and r0 [D]")
            rc = self._L.pumitally_set_point_detectors(self._h, p.ctypes.data_as(_dp), p.size // 3, r.ctypes.data_as(_dp))
        if rc:
            raise ValueError("set_point_detectors failed")

    @property
    def point_detectors(self) -> int:
        """Number of point detectors D, 0 without."""
        return int(self._L.pumitally_get_point_detectors(self._h))

    def set_detector_void(self, on):
        """``on`` True treats the space outside the mesh as a void the detector rays cross: detectors may lie anywhere,
        events outside the mesh are traced, and rays re-enter across concave parts of the hull.  Setting the current
        mode changes nothing; switching resets the tally and discards the folded batches, and switching off while a
        detector lies outside the mesh is refused.  Before comm_init."""
        if self._L.pumitally_set_detector_void(self._h, int(on)):  # anything but 0 or 1 (or a bool) is refused
            raise ValueError("set_detector_void failed")

    @property
    def detector_void(self) -> bool:
        """Whether the space outside the mesh is a void the detector rays cross (set_detector_void)."""
        return bool(self._L.pumitally_get_detector_void(self._h))

    @property
    def detector_hull_entries(self) -> int:
        """Entries of detector rays into the mesh through the hull since the last reset (0 with the void off)."""
        return int(self.get_option("detector_hull_entries"))

    def set_detector_cross_sections(self, sigma):
        """Sigma_t [nbins, num_elements] (caller's numbering, finite, >= 0) the detector rays are attenuated by; the
        score bin is the energy group."""
        s = _host_f64(sigma, "sigma")
        if self._L.pumitally_set_detector_cross_sections(self._h, s.ctypes.data_as(_dp), s.size):
            raise ValueError("set_detector_cross_sections failed")

    def tally_detectors(self, points, weights, pdf=None, responses=None, bins=None, times=None, speeds=None):
        """Events at ``points`` [n, 3], each located as locate() does, scored at every detector: pdf [n, D] per
        steradian (None: isotropic), responses [n, nscores], bins [n], and with time bins times and speeds [n]."""
        p, n = self._points(points)
        _keep, (w, r, b, t, q, v) = self._event_args(n, weights, responses, bins, times, pdf, speeds)
        if self._L.pumitally_tally_detectors(self._h, p.ctypes.data_as(_dp), n, w, q, r, b, t, v):
            raise RuntimeError("tally_detectors failed")

    def tally_detectors_device(self, points, weights, pdf=None, responses=None, bins=None, times=None, speeds=None,
                               stream=None):
        """tally_detectors() on CUDA tensors; enqueued on ``stream`` (default: the current torch stream)."""
        import torch

        if not (points.is_cuda and points.dtype == torch.float64 and points.is_contiguous() and points.numel() % 3 == 0):
            raise TypeError("points must be a contiguous float64 CUDA tensor of shape [n, 3]")
        n = points.numel() // 3
        (w, r, b, t, q, v), stream = self._device_event_args(n, weights, responses, bins, times, stream, points.device,
                                                             pdf, speeds)
        if self._L.pumitally_tally_detectors_device(self._h, points.data_ptr(), n, w, q, r, b, t, v, stream):
            raise RuntimeError("tally_detectors_device failed")

    def tally_detectors_at_particles(self, flagged, weights, pdf=None, responses=None, bins=None, times=None,
                                     speeds=None):
        """Events at the stored positions of the particles i with flagged[i] != 0, in their elements."""
        c = np.ascontiguousarray(flagged, dtype=np.int8).reshape(-1)
        _keep, (w, r, b, t, q, v) = self._event_args(c.size, weights, responses, bins, times, pdf, speeds)
        if self._L.pumitally_tally_detectors_at_particles(self._h, c.ctypes.data_as(_bp), w, q, r, b, t, v, c.size):
            raise RuntimeError("tally_detectors_at_particles failed")

    def tally_detectors_at_particles_device(self, flagged, weights, pdf=None, responses=None, bins=None, times=None,
                                            speeds=None, stream=None):
        """tally_detectors_at_particles() on CUDA tensors (flagged int8 [num_particles]); enqueued on ``stream``."""
        import torch

        n = self.num_particles
        c = self._tensor_ptr(flagged, torch.int8, n, "flagged")
        (w, r, b, t, q, v), stream = self._device_event_args(n, weights, responses, bins, times, stream,
                                                             flagged.device, pdf, speeds)
        if self._L.pumitally_tally_detectors_at_particles_device(self._h, c, w, q, r, b, t, v, n, stream):
            raise RuntimeError("tally_detectors_at_particles_device failed")

    def detector_results(self, kind=0):
        """kind 0 the open tally / per-source divisor, 1 batch mean, 2 standard error, 3 relative error:
        [ntime, nbins, nscores, D]."""
        out = np.empty((max(self.time_bins, 1), self.score_bins, self.scores, self.point_detectors))
        if self._L.pumitally_get_detector_results(self._h, int(kind), out.ctypes.data_as(_dp), out.size):
            raise RuntimeError(f"get_detector_results({kind}) failed")
        return out

    # ---- batch statistics ----------------------------------------------------------
    def set_batch_statistics(self, on: bool):
        """True: keep a running mean and variance of every reported result over batches, on the device (resets the
        tally, discards folded batches); False frees them."""
        if self._L.pumitally_set_batch_statistics(self._h, int(on)):
            raise ValueError("set_batch_statistics failed")

    @property
    def batch_statistics(self) -> bool:
        return bool(self.get_option("batch_statistics"))

    @property
    def batches(self) -> int:
        """Batches folded into the statistics."""
        return self.get_option("batches")

    def end_batch(self):
        """Fold the open batch's per-source results into the statistics and start the next batch (collective with
        several ranks)."""
        if self._L.pumitally_end_batch(self._h):
            raise RuntimeError("end_batch failed")

    def batch_results(self, tally=0, kind=0):
        """tally 0 track length, 1 collision; kind 0 mean, 1 standard error, 2 relative error
        ([ntime, nbins, nscores, num_elements]), 3 gradient of the mean ([..., 3])."""
        shape = (max(self.time_bins, 1), self.score_bins, self.scores, self.num_elements) + ((3,) if kind == 3 else ())
        out = np.empty(shape)
        if self._L.pumitally_get_batch_results(self._h, int(tally), int(kind), out.ctypes.data_as(_dp), out.size):
            raise RuntimeError(f"get_batch_results({tally}, {kind}) failed")
        return out

    def batch_max_rel_err(self, tally=0, score=0):
        """(largest relative error of score ``score`` over the results with a nonzero mean, how many there are)."""
        mx, cnt = C.c_double(0.0), C.c_int64(0)
        if self._L.pumitally_get_batch_max_rel_err(self._h, int(tally), int(score), C.byref(mx), C.byref(cnt)):
            raise RuntimeError(f"get_batch_max_rel_err({tally}, {score}) failed")
        return mx.value, cnt.value

    # ---- region tallies ------------------------------------------------------------
    def set_regions(self, region_of_element, nregions=None):
        """Group the elements into regions: region_of_element[e] in [-1, nregions) for every element (caller's
        numbering; -1: in no region).  nregions None: max + 1.  None as the map removes the regions.  Resets the
        tally and discards the folded batches."""
        if region_of_element is None:
            rc = self._L.pumitally_set_regions(self._h, None, 0, 0)
        else:
            m = np.ascontiguousarray(region_of_element, dtype=np.int32).reshape(-1)
            if nregions is None:
                nregions = int(m.max()) + 1 if m.size else 0
            rc = self._L.pumitally_set_regions(self._h, m.ctypes.data_as(_ip), m.size, int(nregions))
        if rc:
            raise ValueError("set_regions failed")

    @property
    def regions(self) -> int:
        """Number of regions, 0 without regions."""
        return int(self._L.pumitally_get_regions(self._h))

    def region_volumes(self):
        out = np.empty(self.regions)
        if self._L.pumitally_get_region_volumes(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_region_volumes failed")
        return out

    def _region_call(self, fn, tally, kind, what):
        out = np.empty((max(self.time_bins, 1), self.score_bins, self.scores, self.regions))
        if fn(self._h, int(tally), int(kind), out.ctypes.data_as(_dp), out.size):
            raise RuntimeError(f"{what}({tally}, {kind}) failed")
        return out

    def region_results(self, tally=0, kind=1):
        """tally 0 track length, 1 collision; kind 0 raw sum over each region, 1 sum / region volume / per-source
        divisor: [ntime, nbins, nscores, nregions]."""
        return self._region_call(self._L.pumitally_get_region_results, tally, kind, "get_region_results")

    def region_batch_results(self, tally=0, kind=0):
        """kind 0 mean, 1 standard error (both / region volume), 2 relative error of the region sums over the
        batches: [ntime, nbins, nscores, nregions]."""
        return self._region_call(self._L.pumitally_get_region_batch_results, tally, kind, "get_region_batch_results")

    # ---- region currents -----------------------------------------------------------
    def set_region_currents(self, on: bool):
        """True (regions set, face currents on) also reports the partial and net current of every ordered pair of
        adjacent regions, -1 for elements in no region and -2 for outside the mesh; False stops it.  Resets the
        tally and discards the folded batches."""
        if self._L.pumitally_set_region_currents(self._h, int(on)):
            raise ValueError("set_region_currents failed")

    @property
    def region_currents(self) -> bool:
        return bool(self._L.pumitally_get_region_currents(self._h))

    def region_current_pairs(self):
        """(from, to): the int32 region ids of every pair, in ascending (from, to) order (empty while region currents
        are off)."""
        n = int(self._L.pumitally_get_region_current_pair_count(self._h))
        a, b = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        if n and self._L.pumitally_get_region_current_pairs(self._h, a.ctypes.data_as(_ip), b.ctypes.data_as(_ip), n):
            raise RuntimeError("get_region_current_pairs failed")
        return a, b

    def region_current_areas(self):
        """The summed face area of every pair."""
        out = np.empty(int(self._L.pumitally_get_region_current_pair_count(self._h)))
        if self._L.pumitally_get_region_current_areas(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_region_current_areas failed")
        return out

    def region_current_results(self, which=0, kind=0):
        """which 0 partial, 1 net current; kind 0 the open tally / per-source divisor, 1 batch mean, 2 standard
        error, 3 relative error: [ntime, nbins, (C,) npairs] (the cosine axis only while cosine bins are set)."""
        P = int(self._L.pumitally_get_region_current_pair_count(self._h))
        out = np.empty((max(self.time_bins, 1), self.score_bins) + self._cosine_axis() + (P,))
        if self._L.pumitally_get_region_current_results(self._h, int(which), int(kind), out.ctypes.data_as(_dp),
                                                        out.size):
            raise RuntimeError(f"get_region_current_results({which}, {kind}) failed")
        return out

    # ---- checkpoints -------------------------------------------------------------
    def save_checkpoint(self, path):
        """Write the tally state (the open batch if anything was tallied since the last reset, the batch statistics,
        the region statistics) and a fingerprint of the configuration to `path`, atomically (path + ".tmp", then a
        rename).  Changes nothing in the engine.  No particle state: after a load, place the particles first."""
        if self._L.pumitally_save_checkpoint(self._h, os.fsencode(os.fspath(path))):
            raise RuntimeError(f"save_checkpoint({path!r}) failed")

    def load_checkpoint(self, path):
        """Replace the tally state with the checkpoint's; the engine must have the configuration it was saved with
        (and the same ranks, after comm_init).  A refusal changes nothing."""
        if self._L.pumitally_load_checkpoint(self._h, os.fsencode(os.fspath(path))):
            raise RuntimeError(f"load_checkpoint({path!r}) failed")

    def merge_checkpoint(self, path):
        """Add the checkpoint's folded batches to this engine's (batch statistics on, the checkpoint saved at a batch
        end).  The open batch is left alone.  A refusal changes nothing."""
        if self._L.pumitally_merge_checkpoint(self._h, os.fsencode(os.fspath(path))):
            raise RuntimeError(f"merge_checkpoint({path!r}) failed")

    # ---- weight windows ------------------------------------------------------------
    def set_weight_windows(self, lower, upper=None):
        """Set the window table: lower and upper [ngroups, num_elements] (caller's numbering; one group may be given as
        [num_elements]).  lower <= 0 means no window; every other entry must be finite with upper > lower.  None as
        lower removes the windows."""
        if lower is None:
            rc = self._L.pumitally_set_weight_windows(self._h, None, None, 0, 0)
        else:
            lo, hi = _host_f64(lower, "lower"), _host_f64(upper, "upper")
            if lo.size != hi.size or lo.size % max(self.num_elements, 1):
                raise TypeError("lower and upper must both hold ngroups * num_elements values")
            ngroups = lo.size // max(self.num_elements, 1)
            rc = self._L.pumitally_set_weight_windows(self._h, lo.ctypes.data_as(_dp), hi.ctypes.data_as(_dp), lo.size,
                                                      ngroups)
        if rc:
            raise ValueError("set_weight_windows failed")

    @property
    def weight_window_groups(self) -> int:
        """Number of energy groups of the window table, 0 without windows."""
        return int(self._L.pumitally_get_weight_window_groups(self._h))

    def weight_windows(self):
        """(lower, upper), each [ngroups, num_elements] in the caller's numbering; (-1, -1) where there is no window."""
        lo, hi = (np.empty((self.weight_window_groups, self.num_elements)) for _ in range(2))
        if self._L.pumitally_get_weight_windows(self._h, lo.ctypes.data_as(_dp), hi.ctypes.data_as(_dp), lo.size):
            raise RuntimeError("get_weight_windows failed")
        return lo, hi

    def generate_weight_windows(self, tally=0, score=0, time_bin=0, ratio=5.0, max_rel_err=float("inf")):
        """Replace the window table by the MAGIC windows of the batch means of (tally, score, time_bin), the score bins
        as energy groups: lower = phi / phimax * 2 / (ratio + 1), upper = lower * ratio where phi > 0 and its relative
        error is <= max_rel_err (collective with several ranks)."""
        if self._L.pumitally_generate_weight_windows(self._h, int(tally), int(score), int(time_bin), float(ratio),
                                                     float(max_rel_err)):
            raise RuntimeError("generate_weight_windows failed")

    def weight_windows_at_particles(self, groups=None):
        """(lower, upper) [num_particles] of each particle's parent element in energy group groups[i] (None: 0)."""
        lo, hi = np.empty(self.num_particles), np.empty(self.num_particles)
        g = None
        if groups is not None:
            g = np.ascontiguousarray(groups, dtype=np.int32).reshape(-1)
            if g.size != self.num_particles:
                raise TypeError("groups must hold one value per particle")
        if self._L.pumitally_get_weight_windows_at_particles(self._h, None if g is None else g.ctypes.data_as(_ip),
                                                             lo.ctypes.data_as(_dp), hi.ctypes.data_as(_dp), lo.size):
            raise RuntimeError("get_weight_windows_at_particles failed")
        return lo, hi

    def weight_windows_at_particles_device(self, groups=None, stream=None, device=None):
        """weight_windows_at_particles() into float64 CUDA tensors (groups: an int32 CUDA tensor or None), enqueued on
        ``stream`` (default: the current torch stream) behind the last move."""
        import torch

        n = self.num_particles
        dev = groups.device if groups is not None else torch.device("cuda", torch.cuda.current_device()
                                                                     if device is None else device)
        g = self._tensor_ptr(groups, torch.int32, n, "groups")
        lo, hi = torch.empty(n, dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.float64, device=dev)
        if stream is None:
            stream = torch.cuda.current_stream(dev).cuda_stream
        if self._L.pumitally_get_weight_windows_at_particles_device(self._h, g, lo.data_ptr(), hi.data_ptr(), n, stream):
            raise RuntimeError("get_weight_windows_at_particles_device failed")
        return lo, hi

    def weight_windows_at_points(self, points, groups=None):
        """(lower, upper) [npts] at ``points`` [npts, 3], each located as locate() does; (-1, -1) outside the mesh."""
        p, npts = self._points(points)
        lo, hi = np.empty(npts), np.empty(npts)
        g = None
        if groups is not None:
            g = np.ascontiguousarray(groups, dtype=np.int32).reshape(-1)
            if g.size != npts:
                raise TypeError("groups must hold one value per point")
        if self._L.pumitally_get_weight_windows_at_points(self._h, p.ctypes.data_as(_dp), npts,
                                                          None if g is None else g.ctypes.data_as(_ip),
                                                          lo.ctypes.data_as(_dp), hi.ctypes.data_as(_dp)):
            raise RuntimeError("get_weight_windows_at_points failed")
        return lo, hi

    def weight_windows_at_points_device(self, points, groups=None, stream=None):
        """weight_windows_at_points() on a contiguous float64 CUDA tensor [npts, 3]: float64 CUDA tensors, enqueued on
        ``stream`` (default: the current torch stream)."""
        import torch

        if not (points.is_cuda and points.dtype == torch.float64 and points.is_contiguous() and points.numel() % 3 == 0):
            raise TypeError("points must be a contiguous float64 CUDA tensor of shape [npts, 3]")
        npts = points.numel() // 3
        g = self._tensor_ptr(groups, torch.int32, npts, "groups")
        lo = torch.empty(npts, dtype=torch.float64, device=points.device)
        hi = torch.empty(npts, dtype=torch.float64, device=points.device)
        if stream is None:
            stream = torch.cuda.current_stream(points.device).cuda_stream
        if self._L.pumitally_get_weight_windows_at_points_device(self._h, points.data_ptr(), npts, g, lo.data_ptr(),
                                                                 hi.data_ptr(), stream):
            raise RuntimeError("get_weight_windows_at_points_device failed")
        return lo, hi

    # ---- mesh source ---------------------------------------------------------------
    def set_source(self, strength, bias=None, per_volume=False):
        """Set the source: strength [ngroups, num_elements] (caller's numbering; one group may be given as
        [num_elements]), times each element's volume with per_volume, sampled in proportion to strength * bias when a
        bias of the same layout is given.  None as strength removes the source.  A refusal changes nothing."""
        if strength is None:
            rc = self._L.pumitally_set_source(self._h, None, None, 0, 0, 0)
        else:
            q = _host_f64(strength, "strength")
            b = None if bias is None else _host_f64(bias, "bias")
            if q.size % max(self.num_elements, 1) or (b is not None and b.size != q.size):
                raise TypeError("strength (and bias) must hold ngroups * num_elements values")
            rc = self._L.pumitally_set_source(self._h, q.ctypes.data_as(_dp), None if b is None else b.ctypes.data_as(_dp),
                                              q.size, q.size // max(self.num_elements, 1), int(bool(per_volume)))
        if rc:
            raise ValueError("set_source failed")

    @property
    def source_groups(self) -> int:
        """Number of energy groups of the source, 0 without one."""
        return int(self._L.pumitally_get_source_groups(self._h))

    @property
    def source_strength(self) -> float:
        """Q: the total unbiased strength (times the volumes with per_volume), by which the caller normalises."""
        q = C.c_double()
        if self._L.pumitally_get_source_strength(self._h, C.byref(q)):
            raise RuntimeError("get_source_strength failed")
        return q.value

    def sample_source(self, n, seed, first=0, place=False):
        """Samples first .. first + n - 1 of ``seed``: (xyz [n, 3], elem [n] (caller's numbering), group [n],
        weight [n]).  place=True (n == num_particles) also makes sample j particle j's position and parent element."""
        n = int(n)
        xyz, w = np.empty((n, 3)), np.empty(n)
        elem, group = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        if self._L.pumitally_sample_source(self._h, int(seed) & ((1 << 64) - 1), int(first), n, xyz.ctypes.data_as(_dp),
                                           elem.ctypes.data_as(_ip), group.ctypes.data_as(_ip), w.ctypes.data_as(_dp),
                                           int(bool(place))):
            raise RuntimeError("sample_source failed")
        return xyz, elem, group, w

    def sample_source_device(self, n, seed, first=0, place=False, stream=None, device=None):
        """sample_source() into CUDA tensors (float64 [n, 3], int32 [n], int32 [n], float64 [n]), enqueued on
        ``stream`` (default: the current torch stream)."""
        import torch

        n = int(n)
        dev = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        xyz, w = torch.empty((n, 3), dtype=torch.float64, device=dev), torch.empty(n, dtype=torch.float64, device=dev)
        elem, group = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2))
        if stream is None:
            stream = torch.cuda.current_stream(dev).cuda_stream
        if self._L.pumitally_sample_source_device(self._h, int(seed) & ((1 << 64) - 1), int(first), n, xyz.data_ptr(),
                                                  elem.data_ptr(), group.data_ptr(), w.data_ptr(), int(bool(place)),
                                                  stream):
            raise RuntimeError("sample_source_device failed")
        return xyz, elem, group, w

    def WriteTallyResults(self, filename=None):
        if filename is not None:
            self._L.pumitally_set_output_name(self._h, str(filename).encode())
        if self._L.pumitally_write_tally_results(self._h):
            raise RuntimeError("WriteTallyResults failed")

    # ---- raw-pointer variants (host pinned buffers / device tensors) -----------
    def move_host_ptr(self, origin_ptr, dest_ptr, flying_ptr, weights_ptr):
        """MoveToNextLocation on raw host addresses (e.g. pinned torch tensors)."""
        rc = self._L.pumitally_move_to_next_location(
            self._h, C.cast(origin_ptr, _dp), C.cast(dest_ptr, _dp), C.cast(flying_ptr, _bp),
            C.cast(weights_ptr, _dp), 3 * self.num_particles)
        if rc:
            raise RuntimeError("MoveToNextLocation failed")

    def copy_initial_position_device(self, d_xyz_ptr, stream=None):
        if self._L.pumitally_copy_initial_position_device(self._h, d_xyz_ptr, 3 * self.num_particles, stream):
            raise RuntimeError("CopyInitialPosition(device) failed")

    def move_device(self, d_origin, d_dest, d_flying, d_weights, stream=None):
        """MoveToNextLocation on device addresses; enqueues on ``stream`` and returns."""
        if self._L.pumitally_move_to_next_location_device(self._h, d_origin, d_dest, d_flying, d_weights,
                                                          3 * self.num_particles, stream):
            raise RuntimeError("MoveToNextLocation(device) failed")

    def set_state_device(self, d_xyz, d_elem, first, count, stream=None):
        if self._L.pumitally_set_state_device(self._h, d_xyz, d_elem, int(first), int(count), stream):
            raise RuntimeError("set_state_device failed")

    def get_state_device(self, d_xyz, d_elem, first, count, stream=None):
        if self._L.pumitally_get_state_device(self._h, d_xyz, d_elem, int(first), int(count), stream):
            raise RuntimeError("get_state_device failed")

    def get_flux_device(self, d_out, stream=None):
        if self._L.pumitally_get_flux_device(self._h, d_out, stream):
            raise RuntimeError("get_flux_device failed")

    def synchronize(self):
        self._L.pumitally_synchronize(self._h)

    # ---- accessors -----------------------------------------------------------
    @property
    def flux(self):
        out = np.empty(self.num_elements)
        if self._L.pumitally_get_flux(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_flux failed")
        return out

    def normalized_flux(self):
        f, v = np.empty(self.num_elements), np.empty(self.num_elements)
        if self._L.pumitally_get_normalized_flux(self._h, f.ctypes.data_as(_dp), v.ctypes.data_as(_dp), f.size):
            raise RuntimeError("get_normalized_flux failed")
        return f, v

    @property
    def elem_ids(self):
        out = np.empty(self.num_particles, dtype=np.int32)
        if self._L.pumitally_get_element_ids(self._h, out.ctypes.data_as(_ip), out.size):
            raise RuntimeError("get_element_ids failed")
        return out

    @property
    def positions(self):
        out = np.empty((self.num_particles, 3))
        if self._L.pumitally_get_positions(self._h, out.ctypes.data_as(_dp), out.size):
            raise RuntimeError("get_positions failed")
        return out

    @property
    def adjacency(self):
        out = np.empty((self.num_elements, 4), dtype=np.int32)
        if self._L.pumitally_get_adjacency(self._h, out.ctypes.data_as(_ip), out.size):
            raise RuntimeError("get_adjacency failed")
        return out

    def stats(self) -> dict:
        s = Stats()
        if self._L.pumitally_get_stats(self._h, C.byref(s)):
            raise RuntimeError("get_stats failed")
        return {k: getattr(s, k) for k, _ in Stats._fields_}

    def debug_order(self):
        out = np.empty(self.num_particles, dtype=np.int32)
        cnt = int(self._L.pumitally_debug_order(self._h, out.ctypes.data_as(_ip), out.size))
        return out[:max(cnt, 0)]

    def reset_tally(self):
        self._L.pumitally_reset_tally(self._h)

    def set_source_normalization(self, mode: int, value: float = 1.0):
        """0 volume only (reference), 1 /num_particles, 2 /value, 3 /total weight of the batch's first tracks."""
        if self._L.pumitally_set_source_normalization(self._h, int(mode), float(value)):
            raise ValueError(f"bad source normalisation mode={mode} value={value}")

    def source_normalization(self) -> float:
        return float(self._L.pumitally_get_source_normalization(self._h))

    def set_option(self, name: str, value: int):
        if self._L.pumitally_set_option(self._h, name.encode(), int(value)):
            raise ValueError(f"bad option {name}={value}")

    def get_option(self, name: str) -> int:
        return int(self._L.pumitally_get_option(self._h, name.encode()))

    # ---- multi-GPU -------------------------------------------------------------
    @staticmethod
    def nccl_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        if load_library().pumitally_nccl_unique_id(buf):
            raise RuntimeError("ncclGetUniqueId failed")
        return bytes(buf)

    def comm_init(self, rank: int, nranks: int, unique_id: bytes):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        if self._L.pumitally_comm_init(self._h, rank, nranks, buf):
            raise RuntimeError("ncclCommInitRank failed")

    def allreduce_tally(self):
        if self._L.pumitally_allreduce_tally(self._h):
            raise RuntimeError("allreduce_tally failed")

    def exchange_tally(self):
        """Batch-end exchange: the quicker of the two below on this mesh, as measured by comm_init."""
        if self._L.pumitally_exchange_tally(self._h):
            raise RuntimeError("exchange_tally failed")

    def reduce_tally_to_owners(self):
        """Batch-end exchange by ncclReduceScatter; the flux accessors gather the shares (collective)."""
        if self._L.pumitally_reduce_tally_to_owners(self._h):
            raise RuntimeError("reduce_tally_to_owners failed")
