// Links libvalida_b200.so (built by `python -m valida_b200.build`: nvcc -gencode arch=compute_90a,code=sm_90a over
// valida_b200/csrc/**).  VALIDA_B200_LIB_DIR names the directory holding it; the default is this repository's
// valida_b200/ directory, two levels above the crate.
use std::env;
use std::path::PathBuf;

fn main() {
    let dir = env::var("VALIDA_B200_LIB_DIR").map(PathBuf::from).unwrap_or_else(|_| {
        PathBuf::from(env::var("CARGO_MANIFEST_DIR").unwrap()).join("../../valida_b200")
    });
    println!("cargo:rustc-link-search=native={}", dir.display());
    println!("cargo:rustc-link-lib=dylib=valida_b200");
    // the library resolves libcudart through its own RUNPATH; a binary needs to find libvalida_b200.so at run time
    println!("cargo:rustc-link-arg=-Wl,-rpath,{}", dir.display());
    println!("cargo:rerun-if-env-changed=VALIDA_B200_LIB_DIR");
    println!("cargo:rerun-if-changed=../../include/valida_b200.h");
}
