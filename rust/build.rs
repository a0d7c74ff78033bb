fn main() {
    // libsnapb200.so is produced by `python __graft_entry__.py` (nvcc, sm_90a)
    let dir = std::env::var("SNAPB200_LIB_DIR").unwrap_or_else(|_| "../rust-snappy_b200".into());
    println!("cargo:rustc-link-search=native={}", dir);
    println!("cargo:rustc-link-lib=dylib=snapb200");
}
