"""Device discovery for the H100 back-end: the counterpart of `cuda_gpus()` in
watsor/detection/devices.py:28-77, with the same precedence rules --
`CUDA_DEVICE` > `~/.cuda_device` > every visible device, nothing at all when no device is visible
(`CUDA_VISIBLE_DEVICES=""`: the CUDA runtime inside libwatsor_b200 honours it, so the count is 0).
pycuda is not needed: the count comes from `wb_device_count()`.  Checked against the reference
generator (run with stand-in pycuda / tensorrt modules) in tests/test_reference_devices.py."""
import os


def _pinned_device():
    """The single device the user pinned, or None.  Mirrors devices.py:53-72: the environment variable
    wins over the dot file; an unreadable or missing file means "not pinned"; anything that is not an
    integer is a TypeError (raised lazily, from inside the generator, like the reference)."""
    value = os.environ.get('CUDA_DEVICE')
    if value is None:
        home = os.environ.get('HOME')
        if home is not None:
            try:
                with open(os.path.join(home, '.cuda_device')) as f:
                    value = f.read().strip()
            except Exception:
                value = None
    if value is None:
        return None
    try:
        return int(value)
    except Exception as e:
        raise TypeError('CUDA device number (CUDA_DEVICE or ~/.cuda_device) must be an integer') from e


def b200_gpus():
    """Yields (device_index, B200ObjectDetector) for every usable device."""
    try:
        from .. import _lib
        from .b200 import B200ObjectDetector
        visible = _lib.device_count()
    except Exception:
        return
    if visible == 0:
        return
    pinned = _pinned_device()
    for device in ([pinned] if pinned is not None else range(visible)):
        yield device, B200ObjectDetector
