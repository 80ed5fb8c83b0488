"""AsymmetricEncryptionScheme surface (R/encryption/mod.rs)."""
