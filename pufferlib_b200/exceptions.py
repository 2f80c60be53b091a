"""Same exception names and meaning as reference pufferlib/exceptions.py."""


class APIUsageError(RuntimeError):
    """Raised when the API is used incorrectly (reference: pufferlib/exceptions.py:5-10)."""

    def __init__(self, message='API usage error.'):
        self.message = message
        super().__init__(self.message)
