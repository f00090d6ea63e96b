"""CPU: the extract entry points refuse a NULL extractor before anything else, so no device is needed.  Their other refusals are in
tests/test_extract_arguments_gpu.py."""
import ctypes as C

from device_frames import FAKE


def test_null_extractor_refused(api):
    L, F = api.lib(), C.c_void_p(FAKE)         # stands for a buffer: never dereferenced by the host
    calls = {
        "mcs_extract": lambda: L.mcs_extract(None, F, 64, 64, 64, F, 64, F, F, F, F, 100, F),
        "mcs_extract_batch": lambda: L.mcs_extract_batch(None, 1, F, 64, 64, 64, F, F, 1, F, F, F, F, F, 100),
        "mcs_extract_batch_device": lambda: L.mcs_extract_batch_device(None, 1, F, 64, 64, 64, F, F, 1, F, F, F, F, F, 100, None),
        "mcs_extract_batch_packed_device": lambda: L.mcs_extract_batch_packed_device(None, 1, F, 64, 64, 64, F, F, 1, F, F, 100, None),
        "mcs_extract_match_stream": lambda: L.mcs_extract_match_stream(None, 2, 1, F, 64, 64, 64, F, F, F, F, F, F, 100, 2, F, F),
        "mcs_extract_match_stream_packed": lambda: L.mcs_extract_match_stream_packed(None, 2, 1, F, 64, 64, 64, F, F, F, F, F, F, 100, 2, F, F,
                                                                                     F, 50, C.c_double(0.9), F, F, F),
    }
    for name, call in calls.items():
        assert call() == api.MCS_ERR_INVALID, name
        assert L.mcs_last_error().decode() == "null argument", name
