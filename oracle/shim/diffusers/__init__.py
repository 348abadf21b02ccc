"""TEST-ONLY minimal stand-in for diffusers==0.25.0 (pinned by the reference's environment.yaml:20; not installable
here). It exists so that the reference's own src/*.py and ip_adapter/*.py execute UNMODIFIED, in place, from
the reference when oracle/make_golden.py pins oracle/unet_ref.py. Only what the SDXL inference path executes is
implemented (SURVEY.md App. C); everything else is a placeholder class. Never imported by the product."""
from ._stubs import stub_getattr

__version__ = "0.25.0+shim"
__getattr__ = stub_getattr(__name__)
