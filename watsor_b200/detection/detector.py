"""`create_object_detectors` / `ObjectDetector` -- the factory and worker the application calls
(watsor/main.py:414-418), re-implemented for a batched accelerator.  Same signature, same
`device_name` / `fps` / `inference_time` attributes (read by `/metrics`, main.py:242-251), same
latch protocol (exactly one `frame.latch.next()` per drained payload, also on failure --
detector.py:111-112), back-end constructed inside the child so that CUDA state is created after
`spawn` (detector.py:84-96).

Differences from watsor/detection/detector.py:102-112: the worker drains every payload that is
already waiting (at most one per camera: `BalancedQueue` holds a 1-slot semaphore per camera,
sync.py:156-166) and hands them to the GPU as ONE batch; the shared-memory frames are page-locked once
(`wb_register_host`) and the ticks are pipelined over up to four library slots (`submit` / `collect`,
`WATSOR_B200_PIPELINE_DEPTH`): while the GPU runs ticks k-2 .. k the worker writes back tick k-3 and drains the
queue for tick k+1 -- the GPU needs several 8-frame batches in flight to be busy.  A frame's latch still advances
exactly once, after its Detection rows are in its header (also when the back-end raises).
"""
from collections import deque
from multiprocessing.sharedctypes import Array
from os import environ, path
from queue import Empty

from numpy import uint8

try:  # dropped into a watsor checkout: build on the reference's own runtime
    from watsor.stream.share import FramesPerSecond, InferenceTime
    from watsor.stream.work import Payload, Work
except ImportError:  # stand-alone
    from ..stream.work import MeanCounter as InferenceTime
    from ..stream.work import Payload, Work
    from ..stream.work import RateCounter as FramesPerSecond

from .b200 import COMPILED_MODEL, MODEL_FILES
from .devices import b200_gpus


def max_windows(camera_configs):
    """The largest number of detection windows of any camera (1 without any): a frame's model images."""
    return max([len((cfg or {}).get('windows') or ()) for cfg in (camera_configs or {}).values()] + [1])


def has_model(model_path):
    return any(path.isfile(path.join(model_path, f)) for f in (COMPILED_MODEL,) + MODEL_FILES)


def create_object_detectors(delegate_class, stop_event, log_queue, frame_queue, frame_buffers, model_path, kwargs=None):
    """One batched detector worker per visible H100 (detector.py:12-55).  There is deliberately no
    CPU fallback here: without a GPU or a model the assertion below fires, as in the reference."""
    detectors = []
    kwargs = {} if kwargs is None else kwargs
    if has_model(model_path):
        for device, clazz in b200_gpus():
            name = 'detector{}'.format(len(detectors) + 1)
            detectors.append(ObjectDetector(delegate_class, name, stop_event, log_queue, frame_queue, frame_buffers,
                                            kwargs={**kwargs, 'detector_class': clazz,
                                                    'detector_args': (model_path, device)}))
    assert len(detectors) > 0, "Failed to create an object detector. " \
                               "Make sure an H100 is visible and model files are provided."
    return detectors


class ObjectDetector(Work):
    def __init__(self, delegate_class, name, stop_event, log_queue, frame_queue_in, frame_buffers, kwargs=None):
        self.__fps = FramesPerSecond()
        self.__inference_time = InferenceTime()
        self.__device_name = Array('c', 255)
        super().__init__(delegate_class, name, stop_event, log_queue, frame_queue_in,
                         args=(stop_event, frame_buffers, self.__fps, self.__inference_time),
                         kwargs={} if kwargs is None else kwargs)

    @property
    def device_name(self):
        return self.__device_name.value

    @property
    def fps(self):
        return self.__fps

    @property
    def inference_time(self):
        return self.__inference_time

    def _run(self, stop_event, log_queue, *args, **kwargs):
        # base-runtime set-up: with the reference runtime this is Spin._run (thread name, the SIGINT no-op handler a
        # spawned process needs so that Ctrl-C reaches the parent's orderly shutdown instead of raising
        # KeyboardInterrupt mid-batch, logger -> queue; ref: watsor/stream/spin.py:51-58, called the same way as
        # ref: watsor/detection/detector.py:85); the stand-in runtime only has the logger part
        base_run = getattr(super(Work, self), '_run', None)
        if base_run is not None:
            base_run(stop_event, log_queue, *args, **kwargs)
        else:
            self._config_logger(log_queue, *args, **kwargs)
        try:
            detector_class = kwargs.get('detector_class')
            detector_args = kwargs.get('detector_args')
            with detector_class(*detector_args) as object_detector:
                self.__device_name.value = str.encode(object_detector.device_name)[:len(self.__device_name) - 1]
                self._logger.debug("{}{} initialized".format(object_detector.__class__.__name__, detector_args))
                self._cameras = {}
                self._in_flight = deque()
                self._depth = 0
                if callable(getattr(object_detector, 'submit', None)) and callable(getattr(object_detector, 'collect', None)):
                    self._depth = max(1, min(int(kwargs.get('pipeline_depth', environ.get('WATSOR_B200_PIPELINE_DEPTH', 4))), 6))
                    frame_buffers = args[2] if len(args) > 2 else {}
                    self._pin_frame_buffers(object_detector, frame_buffers)
                try:
                    self._spin(self._process, stop_event, *args, object_detector, **kwargs)
                finally:
                    while self._in_flight:              # nothing stays in DETECT state behind us
                        self._collect_oldest(object_detector, *args[3:5])
        except FileNotFoundError as e:
            self._logger.error(e)
        except Exception:
            self._logger.exception('Detection failure')

    def _pin_frame_buffers(self, object_detector, frame_buffers):
        """Page-lock the shared-memory images (ref: watsor/stream/share.py:76-113 allocates them as
        multiprocessing Arrays) so that the H2D copies of a tick are asynchronous DMA transfers."""
        register = getattr(object_detector, 'register_frame_buffer', None)
        if not callable(register):
            return
        buffers = frame_buffers.values() if hasattr(frame_buffers, 'values') else frame_buffers
        for fb in buffers:
            try:
                register(fb)
            except Exception as e:          # pinning is an optimisation: pageable copies still work
                self._logger.warning('could not pin a frame buffer: {}'.format(e))

    # -- one tick: take the payloads that are waiting (block only when the GPU has nothing to do), submit them as
    #    one batch on a free slot, then collect the oldest batch in flight: H2D + kernels of tick k overlap the
    #    result write-back / latch hand-over of tick k-1 and the queue drain of tick k+1
    def _process(self, frame_queue, *args, **kwargs):
        object_detector = args[-1]
        # max_batch counts model images: a camera with detection windows makes one per window
        limit = max(1, getattr(object_detector, 'max_batch', 1) // max_windows(kwargs.get('camera_configs')))
        payloads = []
        busy = bool(getattr(self, '_in_flight', None))
        try:
            first = frame_queue.get_nowait() if busy else frame_queue.get(timeout=1)
            if first is not None:
                payloads.append(first)
        except Empty:
            pass
        while payloads and len(payloads) < limit:
            try:
                nxt = frame_queue.get_nowait()
            except Empty:
                break
            if nxt is not None:
                payloads.append(nxt)
        if payloads:
            self._next_frames(payloads, *args, **kwargs)
        if busy and (not payloads or len(self._in_flight) >= self._depth):
            self._collect_oldest(object_detector, *args[2:4])

    def _next_frame(self, payload, *args, **kwargs):         # single-payload entry of the base class
        self._next_frames([payload], *args, **kwargs)

    def _next_frames(self, payloads, stop_event, frame_buffers, fps, inference_time, object_detector, *args, **kwargs):
        frames = [frame_buffers[p.sender].frames[p.frame_index] for p in payloads]
        handed_over = False
        try:
            if getattr(self, '_depth', 0) > 0 or callable(getattr(object_detector, 'detect_batch', None)):
                images, cams, rows = [], [], []
                for p, frame in zip(payloads, frames):
                    shape, image_np = frame.get_numpy_image(uint8)
                    images.append(image_np)
                    cams.append(self._camera_id(object_detector, p.sender, shape, kwargs.get('camera_configs')))
                    rows.append(frame.header.detections)
                # fuse_filters stays off: the sieve thread applies (and zone-marks) the predicates itself
                if getattr(self, '_depth', 0) > 0:
                    while len(self._in_flight) >= self._depth:
                        self._collect_oldest(object_detector, fps, inference_time)
                    used = {t[0] for t in self._in_flight}
                    slot = next(s for s in range(self._depth) if s not in used)
                    object_detector.submit(slot, images, cams, fuse_filters=False)
                    self._in_flight.append((slot, frames, rows))
                    handed_over = True                       # the latch moves when the batch is collected
                else:
                    ms = object_detector.detect_batch(images, cams, rows, fuse_filters=False)
                    for _ in payloads:
                        inference_time(value=ms)
                        fps(value=True)
            else:                                            # any reference-protocol back-end
                for frame in frames:
                    shape, image_np = frame.get_numpy_image(uint8)
                    inference_time(value=object_detector.detect(shape, image_np, frame.header.detections))
                    fps(value=True)
        finally:
            if not handed_over:
                for frame in frames:
                    if getattr(frame, 'latch', None) is not None:
                        frame.latch.next()

    def _collect_oldest(self, object_detector, fps, inference_time):
        """Wait for the oldest batch in flight, let the library write its Detection rows into the frames' headers,
        update the metrics and advance every frame's latch exactly once (ref: detector.py:111-112 `finally`)."""
        slot, frames, rows = self._in_flight.popleft()
        try:
            ms = object_detector.collect(slot, rows)
            for _ in frames:
                inference_time(value=ms)
                fps(value=True)
        finally:
            for frame in frames:
                if getattr(frame, 'latch', None) is not None:
                    frame.latch.next()

    def _camera_id(self, object_detector, sender, shape, camera_configs):
        key = (sender, int(shape[0]), int(shape[1]))          # a camera that changes its frame size gets a new table
        cam = self._cameras.get(key)
        if cam is None:
            cam = len(self._cameras)
            cfg = (camera_configs or {}).get(sender)
            object_detector.configure_camera(cam, int(shape[1]), int(shape[0]), cfg)
            self._cameras[key] = cam
        return cam
