class VideoProcessor:
    """A video processor: called with a list of frames, returns a list of frames (diffsynth/processors/base.py)."""

    def __init__(self):
        pass

    def __call__(self):
        raise NotImplementedError
