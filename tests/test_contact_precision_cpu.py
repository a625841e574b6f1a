"""Host-side checks of the contact classifier's precision option (no GPU needed: the name is validated first)."""
import pytest


def test_unknown_precision_is_rejected(chd):
    with pytest.raises(ValueError):
        chd.contact.ContactNet({}, precision="bf16")
    with pytest.raises(ValueError):
        chd.contact.detect_contacts("/nonexistent", "/nonexistent", {}, precision="tf32")
    assert chd.contact.precision_code("fp32") == 0 and chd.contact.precision_code("tf32x3") == 1
