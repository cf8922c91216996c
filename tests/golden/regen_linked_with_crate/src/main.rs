//! Writes `<corpus>.linked_<block size id>_<flags>.frame.lz4` for the corpora of lz4_flex's benches: whole frames of
//! `FrameEncoder::with_frame_info(info, Vec::new())`, `write_all`, `finish` with `BlockMode::Linked`, for every block
//! size (0 = Auto, 4..7) and every flag set (bit 0 block checksums, bit 1 content checksum, bit 2 content size).
//! Usage: cargo run --release -- <lz4_flex/benches> <out dir>
use std::fs;
use std::io::Write;
use std::path::Path;

use lz4_flex::frame::{BlockMode, BlockSize, FrameEncoder, FrameInfo};

fn linked_frame(input: &[u8], block_size_id: u32, flags: u32) -> Vec<u8> {
    let bs = match block_size_id {
        4 => BlockSize::Max64KB,
        5 => BlockSize::Max256KB,
        6 => BlockSize::Max1MB,
        7 => BlockSize::Max4MB,
        _ => BlockSize::Auto,
    };
    let mut info = FrameInfo::new().block_size(bs).block_mode(BlockMode::Linked);
    info = info.block_checksums(flags & 1 != 0).content_checksum(flags & 2 != 0);
    if flags & 4 != 0 {
        info = info.content_size(Some(input.len() as u64));
    }
    let mut enc = FrameEncoder::with_frame_info(info, Vec::new());
    enc.write_all(input).unwrap();
    enc.finish().unwrap()
}

fn main() {
    let args: Vec<String> = std::env::args().collect();
    let benches = Path::new(&args[1]);
    let out = Path::new(&args[2]);
    fs::create_dir_all(out).unwrap();
    for f in ["compression_1k.txt", "compression_34k.txt", "compression_66k_JSON.txt", "dickens.txt", "hdfs.json"] {
        let data = fs::read(benches.join(f)).unwrap();
        for bsid in [0u32, 4, 5, 6, 7] {
            for flags in 0u32..8 {
                fs::write(out.join(format!("{f}.linked_{bsid}_{flags}.frame.lz4")), linked_frame(&data, bsid, flags))
                    .unwrap();
            }
        }
    }
    println!("wrote the crate's linked frames to {}", out.display());
}
