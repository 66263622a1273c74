// decoder_sharpen_test.cpp -- the Decoder mirror's batched decode_fountain with should_preprocess chosen per frame (the cimbar
// CLI's decode loop over Extractor results, cimbar.cpp:124-160) against the loop it replaces: single-frame decode_fountain calls on
// one Decoder with the same per-frame flags, in order.
// Usage: decoder_sharpen_test <mode> <frames.rgb> <pattern> <out_prefix>
//   frames.rgb: n raw RGB8 frames of the mode's image size back to back; pattern: n characters '0' / '1' (should_preprocess)
//   writes <out_prefix>.chunks_cc2: the chunks of the batched call under color_correction 2, for the python driver
#include "../../libcimbar_b200/host/Decoder.h"

#include <cstdio>
#include <cstring>
#include <fstream>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

using namespace cb200;

class escrow_buffer_writer   // test-local collector: one buffer slot per write of exactly chunk_size bytes
{
public:
	escrow_buffer_writer(unsigned char* space, unsigned slots, unsigned slot_bytes) : _space(space), _slots(slots), _slotBytes(slot_bytes) {}
	bool good() const { return _ok; }
	unsigned chunk_size() const { return _slotBytes; }
	long tellp() const { return (long)_used * _slotBytes; }
	escrow_buffer_writer& write(const char* data, unsigned length)
	{
		_ok = _ok and length == _slotBytes and _used < _slots;
		if (_ok) { std::memcpy(_space + (size_t)_used * _slotBytes, data, length); ++_used; }
		return *this;
	}
private:
	unsigned char* _space; unsigned _slots, _slotBytes, _used = 0; bool _ok = true;
};

static int fails = 0;
#define CHECK(cond) do { if (!(cond)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #cond); ++fails; } } while (0)

struct Result
{
	std::vector<unsigned char> bytes;
	unsigned good = 0;
	bool has_ccm = false;
	float ccm[9] = {0};
};

// one Decoder, starting without a CCM: the frames one by one, or all of them in one batched call
static Result run(bool use_ecc, bool batched, const std::vector<Image>& imgs, const bool* pre, int cc)
{
	const unsigned n = (unsigned)imgs.size(), cs = cimbar::Config::fountain_chunk_size();
	const unsigned slots = n * (cimbar::Config::capacity() / cs + 1);
	Result r;
	r.bytes.assign((size_t)slots * cs, 0);
	Decoder d(use_ecc);
	d.clear_color_correction();
	escrow_buffer_writer w(r.bytes.data(), slots, cs);
	if (batched) r.good = d.decode_fountain(imgs.data(), n, w, pre, cc);
	else
		for (unsigned f = 0; f < n; ++f) r.good += d.decode_fountain(imgs[f], w, pre[f], cc);
	r.has_ccm = d.get_ccm(r.ccm);
	d.clear_color_correction();
	return r;
}

static void same(const Result& a, const Result& b)
{
	CHECK(a.good == b.good);
	CHECK(std::memcmp(a.bytes.data(), b.bytes.data(), a.good) == 0);
	CHECK(a.has_ccm == b.has_ccm and (!a.has_ccm or std::memcmp(a.ccm, b.ccm, sizeof(a.ccm)) == 0));
}

int main(int argc, char** argv)
{
	if (argc < 5) { std::printf("usage: decoder_sharpen_test <mode> <frames.rgb> <pattern> <out_prefix>\n"); return 2; }
	cimbar::Config::update(std::atoi(argv[1]));
	std::ifstream f(argv[2], std::ios::binary);
	std::vector<unsigned char> pix((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
	const std::string pattern = argv[3], prefix = argv[4];
	const unsigned n = (unsigned)pattern.size();
	const size_t frame_bytes = (size_t)cimbar::Config::image_size_x() * cimbar::Config::image_size_y() * 3;
	CHECK(pix.size() == n * frame_bytes);
	if (pix.size() != n * frame_bytes) return 1;
	std::vector<Image> imgs(n);
	std::unique_ptr<bool[]> pre(new bool[n]);
	for (unsigned k = 0; k < n; ++k)
	{
		imgs[k].rows = cimbar::Config::image_size_y(); imgs[k].cols = cimbar::Config::image_size_x(); imgs[k].data = pix.data() + k * frame_bytes;
		pre[k] = pattern[k] == '1';
	}

	// with ECC and color_correction 2: the fitted CCM carries from frame to frame in order
	Result loop2 = run(true, false, imgs, pre.get(), 2), batch2 = run(true, true, imgs, pre.get(), 2);
	same(loop2, batch2);
	std::ofstream(prefix + ".chunks_cc2", std::ios::binary).write(reinterpret_cast<const char*>(batch2.bytes.data()), batch2.good);
	// with ECC and color_correction 0 / 1
	for (int cc : {0, 1}) same(run(true, false, imgs, pre.get(), cc), run(true, true, imgs, pre.get(), cc));
	// Decoder(use_ecc = false): the raw bit streams, color_correction 1 (the decoder keeps the last frame's matrix)
	same(run(false, false, imgs, pre.get(), 1), run(false, true, imgs, pre.get(), 1));
	same(run(false, false, imgs, pre.get(), 0), run(false, true, imgs, pre.get(), 0));
	// a null flag array is refused
	{
		std::vector<unsigned char> space(cimbar::Config::fountain_chunk_size());
		escrow_buffer_writer w(space.data(), 1, cimbar::Config::fountain_chunk_size());
		bool threw = false;
		try { Decoder().decode_fountain(imgs.data(), n, w, static_cast<const bool*>(nullptr)); }
		catch (const std::invalid_argument&) { threw = true; }
		CHECK(threw);
	}
	std::printf(fails ? "decoder_sharpen_test: %d failure(s)\n" : "decoder_sharpen_test: ok\n", fails);
	return fails ? 1 : 0;
}
