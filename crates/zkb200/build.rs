// Links libzkb200.so (built by `make -C proof_systems_b200/csrc`, nvcc -gencode arch=compute_90a,code=sm_90a).
// ZKB200_LIB_DIR: directory holding libzkb200.so (default: ../../proof_systems_b200 relative to this crate).
use std::{env, path::PathBuf};

fn main() {
    let dir = env::var("ZKB200_LIB_DIR").map(PathBuf::from).unwrap_or_else(|_| {
        PathBuf::from(env::var("CARGO_MANIFEST_DIR").unwrap()).join("../../proof_systems_b200")
    });
    println!("cargo:rustc-link-search=native={}", dir.display());
    println!("cargo:rustc-link-lib=dylib=zkb200");
    println!("cargo:rustc-link-arg=-Wl,-rpath,{}", dir.display());
    println!("cargo:rerun-if-env-changed=ZKB200_LIB_DIR");
    println!("cargo:rerun-if-changed=../../include/zkb200.h");
}
