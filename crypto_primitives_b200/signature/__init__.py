"""SignatureScheme surface (R/signature/mod.rs:14-50)."""
