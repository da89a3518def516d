class Path:
    def __init__(self, *args, **kwargs):
        raise NotImplementedError("matplotlib is not installed")
