"""QuartzNet CTC model package (`Model`, `basecall` are what `load_symbol` looks up for `package = "bonito.ctc"`)."""
from bonito_b200.ctc.model import Model  # noqa: F401
from bonito_b200.ctc.basecall import basecall  # noqa: F401
