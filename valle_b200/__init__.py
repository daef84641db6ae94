"""valle_b200 -- H100-native (sm_90a) VALL-E decoding engine behind the reference's
`valle.models.VALLE` / `valle.modules` API.  See DESIGN.md / INTEGRATION.md."""
__version__ = "0.1.0"
