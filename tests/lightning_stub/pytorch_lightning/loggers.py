"""`pytorch_lightning.loggers` of the test stand-in: a placeholder `Logger` (rectools/models/nn/dssm.py imports it)."""


class Logger:
    """Placeholder: nothing is logged."""
