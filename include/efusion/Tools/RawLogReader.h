// Headless .klg reader for programs written against the reference's Tools/LogReader interface
// (reference Tools/LogReader.h:32-88, Tools/RawLogReader.h:35-66): same public members (timestamp, depth, rgb,
// currentFrame, flipColors) and methods (getNext, getBack, hasMore, rewind, rewound, fastForward, getNumFrames, getFile,
// setAuto), so the frame loop of MainController.cpp:216-245 compiles unchanged against it.
//
// File layout (Tools/RawLogReader.cpp:22-109): int32 numFrames; per frame int64 timestamp, int32 depthSize,
// int32 imageSize, depth payload, image payload. depthSize == 2*W*H / imageSize == 3*W*H mark raw payloads; a smaller
// depth payload is zlib-compressed (supported when <zlib.h> is available, link with -lz); a smaller non-empty image
// payload is JPEG, decoded by Tools/JPEGLoader.h (own baseline decoder, bit-identical to libjpeg's default output).
// hasMore() keeps the reference's "currentFrame + 1 < numFrames" (the last frame of a log is never delivered,
// RawLogReader.cpp:139-141).
//
// Addition: peekNext() decodes the frame AFTER the current one into a second buffer pair without advancing, so the
// caller can hand it to ElasticFusion::processFrame(..., nextRgb, nextDepth) for the look-ahead; the following getNext()
// just flips the buffers.
#ifndef EFUSION_B200_RAWLOGREADER_H_
#define EFUSION_B200_RAWLOGREADER_H_

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stack>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../Utils/Resolution.h"
#include "JPEGLoader.h"

#if defined(__has_include)
#if __has_include(<zlib.h>) && !defined(EFUSION_NO_ZLIB)
#include <zlib.h>
#define EFUSION_HAVE_ZLIB 1
#endif
#endif

class LogReader {
 public:
  LogReader(std::string file, bool flipColors)
      : flipColors(flipColors), timestamp(0), depth(nullptr), rgb(nullptr), currentFrame(0), file_(std::move(file)),
        width_(Resolution::getInstance().width()), height_(Resolution::getInstance().height()), numPixels_(width_ * height_) {}
  virtual ~LogReader() {}
  virtual void getNext() = 0;
  virtual int getNumFrames() = 0;
  virtual bool hasMore() = 0;
  virtual bool rewound() = 0;
  virtual void rewind() = 0;
  virtual void getBack() = 0;
  virtual void fastForward(int frame) = 0;
  virtual const std::string getFile() = 0;
  virtual void setAuto(bool value) = 0;

  bool flipColors;
  int64_t timestamp;
  uint16_t* depth;
  uint8_t* rgb;
  int currentFrame;

 protected:
  const std::string file_;
  int width_, height_, numPixels_;
};

class RawLogReader : public LogReader {
 public:
  RawLogReader(std::string file, bool flipColors) : LogReader(std::move(file), flipColors) {
    for (int s = 0; s < 2; ++s) {
      depthBuf_[s].resize((size_t)numPixels_);
      rgbBuf_[s].resize((size_t)numPixels_ * 3);
    }
    open();
  }
  ~RawLogReader() override {
    if (fp_) std::fclose(fp_);
  }

  void getNext() override {
    filePointers.push(frameStart_);
    if (peeked_) {  // already decoded by peekNext(): flip the buffers, the file position is past that frame
      cur_ ^= 1;
      timestamp = peekTimestamp_;
      peeked_ = false;
      frameStart_ = std::ftell(fp_);
    } else {
      readFrame(cur_, timestamp);
      frameStart_ = std::ftell(fp_);
    }
    publish();
    currentFrame++;
  }

  // Decodes the frame that the next getNext() will deliver (no state visible through the LogReader interface changes).
  // Returns false when the log has no further frame to deliver.
  bool peekNext() {
    if (peeked_) return true;
    if (!hasMore()) return false;
    readFrame(cur_ ^ 1, peekTimestamp_);
    peeked_ = true;
    return true;
  }
  const uint8_t* nextRgb() const { return peeked_ ? rgbBuf_[cur_ ^ 1].data() : nullptr; }
  const uint16_t* nextDepth() const { return peeked_ ? depthBuf_[cur_ ^ 1].data() : nullptr; }
  int64_t nextTimestamp() const { return peekTimestamp_; }

  void getBack() override {
    if (filePointers.empty()) throw std::runtime_error("RawLogReader::getBack: nothing to go back to");
    dropPeek();
    std::fseek(fp_, filePointers.top(), SEEK_SET);
    filePointers.pop();
    readFrame(cur_, timestamp);
    frameStart_ = std::ftell(fp_);
    publish();
    currentFrame++;  // (the reference's getCore increments here as well, RawLogReader.cpp:104)
  }

  int getNumFrames() override { return numFrames_; }
  bool hasMore() override { return currentFrame + 1 < numFrames_; }
  bool rewound() override { return filePointers.empty(); }

  void rewind() override {
    std::stack<long> empty;
    std::swap(empty, filePointers);
    dropPeek();
    std::fclose(fp_);
    fp_ = nullptr;
    open();
  }

  void fastForward(int frame) override {
    dropPeek();
    while (currentFrame < frame && hasMore()) {
      filePointers.push(std::ftell(fp_));
      int64_t ts;
      int32_t dsz, isz;
      readHeader(ts, dsz, isz);
      std::fseek(fp_, (long)dsz + (long)(isz > 0 ? isz : 0), SEEK_CUR);
      timestamp = ts;
      currentFrame++;
    }
    frameStart_ = std::ftell(fp_);
  }

  const std::string getFile() override { return file_; }
  void setAuto(bool) override {}

  std::stack<long> filePointers;

 private:
  void open() {
    fp_ = std::fopen(file_.c_str(), "rb");
    if (!fp_) throw std::runtime_error("RawLogReader: cannot open " + file_);
    if (std::fread(&numFrames_, sizeof(int32_t), 1, fp_) != 1) throw std::runtime_error("RawLogReader: empty log " + file_);
    currentFrame = 0;
    frameStart_ = std::ftell(fp_);
    peeked_ = false;
    cur_ = 0;
  }
  void dropPeek() {
    if (peeked_) {
      std::fseek(fp_, frameStart_, SEEK_SET);
      peeked_ = false;
    }
  }
  void readHeader(int64_t& ts, int32_t& dsz, int32_t& isz) {
    if (std::fread(&ts, sizeof(int64_t), 1, fp_) != 1 || std::fread(&dsz, sizeof(int32_t), 1, fp_) != 1 ||
        std::fread(&isz, sizeof(int32_t), 1, fp_) != 1 || dsz < 0 || isz < 0)
      throw std::runtime_error("RawLogReader: truncated frame header in " + file_);
  }
  void readFrame(int slot, int64_t& ts) {
    int32_t dsz, isz;
    readHeader(ts, dsz, isz);
    uint16_t* d = depthBuf_[slot].data();
    uint8_t* c = rgbBuf_[slot].data();
    if (dsz == numPixels_ * 2) {
      if (std::fread(d, 1, (size_t)dsz, fp_) != (size_t)dsz) throw std::runtime_error("RawLogReader: truncated depth payload");
    } else {
      scratch_.resize((size_t)dsz);
      if (dsz && std::fread(scratch_.data(), 1, (size_t)dsz, fp_) != (size_t)dsz) throw std::runtime_error("RawLogReader: truncated depth payload");
#ifdef EFUSION_HAVE_ZLIB
      unsigned long len = (unsigned long)numPixels_ * 2;
      if (uncompress(reinterpret_cast<Bytef*>(d), &len, reinterpret_cast<const Bytef*>(scratch_.data()), (unsigned long)dsz) != Z_OK)
        throw std::runtime_error("RawLogReader: zlib depth payload does not decompress");
#else
      throw std::runtime_error("RawLogReader: zlib-compressed depth payload (build with zlib)");
#endif
    }
    if (isz == numPixels_ * 3) {
      if (std::fread(c, 1, (size_t)isz, fp_) != (size_t)isz) throw std::runtime_error("RawLogReader: truncated image payload");
    } else if (isz > 0) {
      jpegBuf_.resize((size_t)isz);
      if (std::fread(jpegBuf_.data(), 1, (size_t)isz, fp_) != (size_t)isz) throw std::runtime_error("RawLogReader: truncated image payload");
      int jw = 0, jh = 0;
      JPEGLoader::decode(jpegBuf_.data(), (size_t)isz, jpegRgb_, jw, jh);
      if (jw != width_ || jh != height_) throw std::runtime_error("RawLogReader: JPEG payload size differs from the log resolution");
      for (int i = 0; i < numPixels_; ++i) {  // JPEGLoader::readData's channel swap (reference Tools/JPEGLoader.h:73-82)
        c[i * 3 + 0] = jpegRgb_[(size_t)i * 3 + 2];
        c[i * 3 + 1] = jpegRgb_[(size_t)i * 3 + 1];
        c[i * 3 + 2] = jpegRgb_[(size_t)i * 3 + 0];
      }
    } else {
      std::memset(c, 0, (size_t)numPixels_ * 3);
    }
    if (flipColors)
      for (int i = 0; i < numPixels_ * 3; i += 3) std::swap(c[i], c[i + 2]);
  }
  void publish() {
    depth = depthBuf_[cur_].data();
    rgb = rgbBuf_[cur_].data();
  }

  FILE* fp_ = nullptr;
  int32_t numFrames_ = 0;
  long frameStart_ = 0;  // file offset of the frame the next getNext() delivers
  std::vector<uint16_t> depthBuf_[2];
  std::vector<uint8_t> rgbBuf_[2];
  std::vector<uint8_t> scratch_, jpegBuf_, jpegRgb_;
  int cur_ = 0;
  bool peeked_ = false;
  int64_t peekTimestamp_ = 0;
};

#endif  // EFUSION_B200_RAWLOGREADER_H_
