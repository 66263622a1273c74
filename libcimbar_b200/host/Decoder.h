// Decoder.h -- header-compatible mirror of libcimbar's Decoder (reference: src/lib/encoder/Decoder.h:16-189).
// Same constructor and the same two templates
//     unsigned decode(const MAT& img, STREAM& ostream, bool should_preprocess=false, int color_correction=2)
//     unsigned decode_fountain(const MAT& img, FOUNTAINSTREAM& ostream, bool should_preprocess=false, int color_correction=2)
// (plus batched decode_fountain overloads over n frames, with one should_preprocess for all of them or one per frame)
// with the same stream protocol and the same return value (good bytes).  The frame is decoded on the GPU through the C ABI;
// the host only hands the results to the caller's stream:
//   decode()           good RS blocks are write()n, failed ones announced with `stream << BadChunk(n)` -- what the two
//                      reed_solomon_streams of Decoder.h:100-117 do with the caller's stream;
//   decode_fountain()  the device has already applied aligned_stream's chunk rule (a chunk is emitted iff all its RS blocks
//                      decoded and the chunk before it did not end in a bad block, aligned_stream.h:39-116; k_chunk_mask), so
//                      the accepted chunks of cb200_decode_fountain are written to the caller's fountain stream one write()
//                      per chunk, exactly the calls the reference's aligned_stream<FOUNTAINSTREAM> would make.
// Stream classes are the caller's own (std::stringstream, std::ofstream, the reference's escrow_buffer_writer /
// fountain_decoder_sink / aligned_stream, cb200::fountain_sink ...): nothing of them is restated here.
//
// BAD is the tag type a failed RS block is announced with; an integrated build instantiates DecoderT<ReedSolomon::BadChunk>
// so that the reference's own operator<< overloads are picked up (INTEGRATION.md).
//
// MAT: anything with .rows, .cols, .channels(), .data, .isContinuous() -- a cv::Mat works, so does cb200::Image.
// Differences from the reference:
//   * frames must be exactly Config::image_size_x() x image_size_y(), RGB8, continuous (the Extractor's output);
//     a smaller image reproduces the reference's degenerate "reader not good" result (zero-filled streams);
//   * color_correction outside 0..2 is decoded as 0 and reported through last_warnings().
// The colour correction matrix is the calling thread's and the device context is cached per (thread, device, mode)
// (detail.h), so building a fresh Decoder per frame -- what cimbar_recv_js.cpp:164 does -- keeps the fitted matrix and costs
// nothing.
#pragma once
#include "../../include/cb200.h"
#include "Config.h"
#include "detail.h"
#include "streams.h"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace cb200 {

struct Image   // minimal cv::Mat-shaped view over caller-owned RGB8 pixels
{
	int rows = 0, cols = 0;
	const unsigned char* data = nullptr;
	int nchannels = 3;
	int channels() const { return nchannels; }
	bool isContinuous() const { return true; }
};

template <typename BAD>
class DecoderT
{
public:
	static const unsigned WARN_COLOR_CORRECTION_IGNORED = 1;

	DecoderT(bool use_ecc = true, bool interleave = true, int device = -1)
		: _useEcc(use_ecc), _interleave(interleave), _device(device), _modeVal(cimbar::Config::mode_val())
	{
		cb200_get_info(ctx(1), &_info);
	}

	unsigned last_warnings() const { return _warnings; }
	unsigned last_frame_flags() const { return _frameFlags; }   // CB200_FRAME_FALLBACK: the exact flood walk was needed

	// The decoder's colour correction matrix: CimbDecoder::update_color_correction / get_ccm (CimbDecoder.cpp:76-85), row-major
	void update_color_correction(const float m9[9])
	{
		detail::ThreadCcm& t = detail::thread_ccm();
		t.active = true;
		std::memcpy(t.m, m9, sizeof(t.m));
		++t.version;
	}
	void clear_color_correction() { detail::thread_ccm().active = false; ++detail::thread_ccm().version; }
	bool get_ccm(float m9[9]) const
	{
		const detail::ThreadCcm& t = detail::thread_ccm();
		if (t.active) std::memcpy(m9, t.m, sizeof(t.m));
		return t.active;
	}
	// DecoderPlus::load_ccm / save_ccm (src/lib/encoder/DecoderPlus.h:31-55): the file is the 9 float32 of the matrix
	bool load_ccm(const std::string& filename)
	{
		FILE* f = fopen(filename.c_str(), "rb");
		if (!f) return false;
		float m[9];
		size_t got = fread(m, 1, sizeof(m), f);
		fclose(f);
		if (got < sizeof(m)) return false;
		update_color_correction(m);
		return true;
	}
	bool save_ccm(const std::string& filename) const
	{
		float m[9];
		if (!get_ccm(m)) return false;
		FILE* f = fopen(filename.c_str(), "wb");
		if (!f) return false;
		size_t put = fwrite(m, 1, sizeof(m), f);
		fclose(f);
		return put == sizeof(m);
	}

	template <typename MAT, typename STREAM>
	unsigned decode(const MAT& img, STREAM& ostream, bool should_preprocess = false, int color_correction = 2)
	{
		return decode_into(img, ostream, should_preprocess, color_correction);
	}

	template <typename MAT, typename FOUNTAINSTREAM>
	unsigned decode_fountain(const MAT& img, FOUNTAINSTREAM& ostream, bool should_preprocess = false, int color_correction = 2)
	{
		const MAT* one = &img;
		return decode_fountain(one, 1, ostream, should_preprocess, color_correction);
	}

	// Batched form of decode_fountain: `n` frames go to the device in ONE call (one H2D copy, one launch sequence, one D2H copy)
	// and their accepted chunks reach the stream frame by frame, in order -- the result of n single-frame calls made by one
	// reference decoder (the CCM carries from frame to frame).  Returns the good bytes of all frames.
	template <typename MAT, typename FOUNTAINSTREAM>
	unsigned decode_fountain(const MAT* imgs, unsigned n, FOUNTAINSTREAM& ostream, bool should_preprocess = false, int color_correction = 2)
	{
		return decode_fountain_batch(imgs, n, ostream, nullptr, should_preprocess, color_correction);
	}

	// The same with should_preprocess chosen per frame (n flags): the cimbar CLI's decode loop (cimbar.cpp:124-160) over
	// cb200::Extractor results -- `should_preprocess[f] = extract(...) == Extractor::NEEDS_SHARPEN` -- in one call.
	template <typename MAT, typename FOUNTAINSTREAM>
	unsigned decode_fountain(const MAT* imgs, unsigned n, FOUNTAINSTREAM& ostream, const bool* should_preprocess, int color_correction = 2)
	{
		if (!should_preprocess) throw std::invalid_argument("cb200::Decoder: null should_preprocess");
		return decode_fountain_batch(imgs, n, ostream, should_preprocess, false, color_correction);
	}

protected:
	// each: n should_preprocess flags, or nullptr = should_preprocess for every frame
	template <typename MAT, typename FOUNTAINSTREAM>
	unsigned decode_fountain_batch(const MAT* imgs, unsigned n, FOUNTAINSTREAM& ostream, const bool* each, bool should_preprocess,
	                               int color_correction)
	{
		const unsigned chunk_size = _info.chunk_size;
		// Decoder.h:180-185: on a chunk-size mismatch the decode is eaten (it still runs, and still updates the CCM)
		const bool deliver = ostream.chunk_size() == chunk_size;
		_warnings = (color_correction < 0 or color_correction > 2) ? WARN_COLOR_CORRECTION_IGNORED : 0;
		_frameFlags = 0;
		check_mode();
		// per frame: the chunks aligned_stream would flush, densely packed, and how many of them
		const size_t per_frame = std::max<size_t>(_info.data_bytes, _info.raw_bytes);
		std::vector<uint8_t> chunks((size_t)n * per_frame);
		std::vector<uint32_t> count(n, 0);
		std::vector<unsigned> good_idx;                  // frames the device decodes (the others are "reader not good")
		for (unsigned f = 0; f < n; ++f)
		{
			if (frame_good(imgs[f])) { check_exact(imgs[f]); good_idx.push_back(f); continue; }
			// zero-filled streams (plus the one colour bit, see degenerate()) still flow through RS and the aligner: every
			// whole chunk of them is flushed to the stream
			std::vector<uint8_t> data, ok;
			degenerate(imgs[f], data, ok);
			count[f] = (uint32_t)(data.size() / chunk_size);
			std::memcpy(chunks.data() + (size_t)f * per_frame, data.data(), (size_t)count[f] * chunk_size);
		}
		if (!good_idx.empty())
		{
			const unsigned m = (unsigned)good_idx.size();
			cb200_ctx* c = ctx((int)m);
			// the C ABI takes one contiguous batch; contiguous inputs (a frame ring) are passed through without a copy
			const uint8_t* batch = imgs[good_idx[0]].data;
			std::vector<uint8_t> packed;
			bool contiguous = true;
			for (unsigned k = 1; k < m; ++k) contiguous = contiguous and imgs[good_idx[k]].data == batch + (size_t)k * _info.frame_bytes;
			if (!contiguous)
			{
				packed.resize((size_t)m * _info.frame_bytes);
				for (unsigned k = 0; k < m; ++k) std::memcpy(packed.data() + (size_t)k * _info.frame_bytes, imgs[good_idx[k]].data, _info.frame_bytes);
				batch = packed.data();
			}
			std::vector<uint8_t> ff(m);
			detail::push_ccm(c);
			// the fit of color_correction 2 needs this stream's chunk callbacks in the reference: they exist in decode_fountain only
			const uint32_t flags = flags_for(each ? false : should_preprocess, color_correction, true);
			std::vector<uint8_t> sel;
			if (each)
				for (unsigned k = 0; k < m; ++k) sel.push_back(each[good_idx[k]] ? 1 : 0);
			if (_useEcc)
			{
				std::vector<uint8_t> out((size_t)m * _info.data_bytes);
				std::vector<uint32_t> cnt(m), mask(m);
				const int rc = each ? cb200_decode_fountain_sharpen(c, batch, (int)m, flags, sel.data(), out.data(), cnt.data(), mask.data(), ff.data())
				                         : cb200_decode_fountain(c, batch, (int)m, flags, out.data(), cnt.data(), mask.data(), ff.data());
				if (rc != CB200_OK)
					throw std::runtime_error(std::string("cb200_decode_fountain: ") + cb200_last_error());
				for (unsigned k = 0; k < m; ++k)
				{
					count[good_idx[k]] = cnt[k];
					std::memcpy(chunks.data() + (size_t)good_idx[k] * per_frame, out.data() + (size_t)k * _info.data_bytes, (size_t)cnt[k] * chunk_size);
				}
			}
			else
			{   // ecc_bytes = 0: the raw bit stream passes through reed_solomon_stream untouched and is re-chunked as it is;
				// the tail that does not fill a chunk is never flushed.  No RS pass means no header for a CCM fit.
				std::vector<uint8_t> raw((size_t)m * _info.raw_bytes);
				if (!each)
				{
					if (cb200_decode_raw(c, batch, (int)m, flags & ~CB200_FLAG_CC_FIT, raw.data(), ff.data()) != CB200_OK)
						throw std::runtime_error(std::string("cb200_decode_raw: ") + cb200_last_error());
				}
				else
				{   // no fit, so nothing carries between frames except the CCM the last one leaves (color_correction 1): one call
					// per kind, the kind of the last frame last
					for (int pass = 0; pass < 2; ++pass)
					{
						const uint8_t kind = (uint8_t)(pass == 0 ? !sel[m - 1] : sel[m - 1]);
						std::vector<unsigned> ks;
						for (unsigned k = 0; k < m; ++k) if (sel[k] == kind) ks.push_back(k);
						if (ks.empty()) continue;
						std::vector<uint8_t> in(ks.size() * (size_t)_info.frame_bytes), part(ks.size() * (size_t)_info.raw_bytes), pff(ks.size());
						for (size_t j = 0; j < ks.size(); ++j) std::memcpy(in.data() + j * _info.frame_bytes, batch + (size_t)ks[j] * _info.frame_bytes, _info.frame_bytes);
						if (cb200_decode_raw(c, in.data(), (int)ks.size(), (flags & ~CB200_FLAG_CC_FIT) | (kind ? CB200_FLAG_SHARPEN : 0u), part.data(), pff.data()) != CB200_OK)
							throw std::runtime_error(std::string("cb200_decode_raw: ") + cb200_last_error());
						for (size_t j = 0; j < ks.size(); ++j)
						{
							std::memcpy(raw.data() + (size_t)ks[j] * _info.raw_bytes, part.data() + j * _info.raw_bytes, _info.raw_bytes);
							ff[ks[j]] = pff[j];
						}
					}
				}
				if (flags & CB200_FLAG_CC_FIT) _warnings |= WARN_COLOR_CORRECTION_IGNORED;
				for (unsigned k = 0; k < m; ++k)
				{
					count[good_idx[k]] = _info.raw_bytes / chunk_size;
					std::memcpy(chunks.data() + (size_t)good_idx[k] * per_frame, raw.data() + (size_t)k * _info.raw_bytes,
					            (size_t)count[good_idx[k]] * chunk_size);
				}
			}
			detail::pull_ccm(c);
			for (unsigned k = 0; k < m; ++k) _frameFlags |= ff[k];
		}
		unsigned total = 0;
		for (unsigned f = 0; f < n; ++f)
			for (unsigned q = 0; q < count[f]; ++q)
			{
				// aligned_stream::write drops everything once the stream below it stops being good (aligned_stream.h:39-44)
				if (deliver and !ostream.good()) return total;
				if (deliver) ostream.write(reinterpret_cast<const char*>(chunks.data()) + (size_t)f * per_frame + (size_t)q * chunk_size, chunk_size);
				total += chunk_size;
			}
		return total;
	}

	cb200_ctx* ctx(int frames) const { return detail::thread_context(_device, _modeVal, frames); }

	void check_mode() const
	{
		if (cimbar::Config::mode_val() != _modeVal)
			throw std::runtime_error("cb200::Decoder: Config mode changed after construction (one Decoder per mode)");
	}
	template <typename MAT>
	bool frame_good(const MAT& img) const
	{   // CimbReader.cpp:119
		return img.cols >= _info.image_size_x and img.rows >= _info.image_size_y and img.channels() == 3;
	}
	template <typename MAT>
	void check_exact(const MAT& img) const
	{
		if (img.cols != _info.image_size_x or img.rows != _info.image_size_y or !img.isContinuous())
			throw std::invalid_argument("cb200::Decoder: frame must be exactly image_size_x x image_size_y, continuous RGB8");
	}
	uint32_t flags_for(bool should_preprocess, int color_correction, bool header_callbacks) const
	{
		return (should_preprocess ? CB200_FLAG_SHARPEN : 0u) | (color_correction == 1 ? CB200_FLAG_CC_SIMPLE : 0u) |
		       ((color_correction == 2 and header_callbacks) ? CB200_FLAG_CC_FIT : 0u) | (_interleave ? 0u : CB200_FLAG_NO_INTERLEAVE);
	}

	// reader not good (undersized image): zero-filled symbol/colour buffers are still flushed (CimbReader.cpp:141-142,
	// Decoder.h:100-117).  Every colorPositions entry is still the default {0,0,0}, so the colour pass ORs the colour decoded at
	// pixel (0,0) into bit position 0 (Decoder.h:107-114 / :153-158); after RS that single byte is corrected back to 0.
	template <typename MAT>
	void degenerate(const MAT& img, std::vector<uint8_t>& data, std::vector<uint8_t>& ok)
	{
		const size_t out_bytes = _useEcc ? (size_t)_info.data_bytes : (size_t)_info.raw_bytes;
		data.assign(out_bytes, 0);
		ok.assign(_info.rs_blocks, 1);
		if (!_useEcc and img.channels() == 3 and img.cols >= 8 and img.rows >= 8 and img.isContinuous())
		{
			unsigned r = 0, g = 0, b = 0;
			for (int i = 1; i <= 6; ++i)
				for (int j = 1; j <= 6; ++j)
				{
					const unsigned char* p = img.data + ((size_t)i * img.cols + j) * 3;
					r += p[0]; g += p[1]; b += p[2];
				}
			uint8_t mean[3] = {(uint8_t)(r / 36), (uint8_t)(g / 36), (uint8_t)(b / 36)}, col = 0;
			cb200_ctx* c = ctx(1);
			detail::push_ccm(c);
			if (cb200_best_colors(c, mean, 1, &col) != CB200_OK)
				throw std::runtime_error(std::string("cb200_best_colors: ") + cb200_last_error());
			size_t at = _info.legacy_mode ? 0 : (size_t)_info.raw_symbol_bytes;
			data[at] |= (uint8_t)(col << (8 - _info.color_bits));
		}
	}
	template <typename MAT, typename STREAM>
	unsigned decode_into(const MAT& img, STREAM& ostream, bool should_preprocess, int color_correction)
	{
		_warnings = (color_correction < 0 or color_correction > 2) ? WARN_COLOR_CORRECTION_IGNORED : 0;
		_frameFlags = 0;
		check_mode();
		std::vector<uint8_t> data, ok;
		if (!frame_good(img)) degenerate(img, data, ok);
		else
		{
			check_exact(img);
			const size_t out_bytes = _useEcc ? (size_t)_info.data_bytes : (size_t)_info.raw_bytes;
			data.assign(out_bytes, 0);
			ok.assign(_info.rs_blocks, 1);
			cb200_ctx* c = ctx(1);
			detail::push_ccm(c);
			// Decoder::decode on a caller's stream has no chunk callbacks: color_correction 2 decodes with the CCM the thread holds
			uint32_t flags = flags_for(should_preprocess, color_correction, false);
			uint8_t ff = 0;
			int rc = _useEcc ? cb200_decode(c, img.data, 1, flags, data.data(), ok.data(), &ff)
			                 : cb200_decode_raw(c, img.data, 1, flags, data.data(), &ff);
			if (rc != CB200_OK) throw std::runtime_error(std::string("cb200 decode: ") + cb200_last_error());
			detail::pull_ccm(c);
			_frameFlags = ff;
		}
		if (!_useEcc)   // reed_solomon_stream pass-through (reed_solomon_stream.h:58-62): the raw cell bits
		{
			ostream.write(reinterpret_cast<const char*>(data.data()), (unsigned)data.size());
			return (unsigned)ostream.tellp();
		}
		// two reed_solomon_streams (symbols, colours) flushing into the same ostream (Decoder.h:100-101, :115-117)
		const unsigned msg = _info.ecc_block_size - _info.ecc_bytes;
		for (int b = 0; b < _info.rs_blocks; ++b)
		{
			if (ok[b]) ostream.write(reinterpret_cast<const char*>(data.data()) + (size_t)b * msg, msg);
			else ostream << BAD(msg);
		}
		return (unsigned)ostream.tellp();
	}

protected:
	bool _useEcc;
	bool _interleave;
	int _device;
	int _modeVal;
	cb200_info _info;
	unsigned _warnings = 0;
	unsigned _frameFlags = 0;
};

using Decoder = DecoderT<BadChunk>;

}  // namespace cb200
