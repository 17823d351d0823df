// JSMpeg.Decoder.MPEG1VideoB200 -- the reference-side binding for libjsmpeg_b200.so.
//
// NOT RUN IN THIS REPOSITORY'S IMAGE (no Node / JS engine; see INTEGRATION.md).  It has the surface
// of JSMpeg.Decoder.MPEG1Video / MPEG1VideoWASM (reference src/mpeg1.js:6-64, src/mpeg1-wasm.js):
// the player picks it exactly where it picks the WASM decoder (src/player.js:35-38), e.g.
//     options.decoderB200 ? new JSMpeg.Decoder.MPEG1VideoB200(options) : ...
// Everything except the five native calls is inherited from JSMpeg.Decoder.Base
// (src/decoder.js): PTS table, seek, advanceDecodedTime, currentTime.
// The host-side mirror that IS tested here is jsmpeg_b200/decoder.py (same logic, Python).

JSMpeg.Decoder.MPEG1VideoB200 = (function(){ "use strict";

var native = require('./jsmpeg_b200.node');

var MPEG1B200 = function(options) {
	JSMpeg.Decoder.Base.call(this, options);
	this.onDecodeCallback = options.onVideoDecode;
	var bufferSize = options.videoBufferSize || 512*1024;
	var bufferMode = options.streaming ? 1 /* EVICT */ : 2 /* EXPAND */;
	this.decoder = native.create(bufferSize, bufferMode);
	// extension: decode B pictures (the reference skips them, src/mpeg1.js:181-184); pictures then arrive in
	// CODED order, native.lastPictureType(this.decoder) tells a renderer which ones to hold back
	if (options.decodeBPictures) { native.setDecodeB(this.decoder, 1); }
	// ... and with displayOrder an I/P picture is held back (a copy: the planes are borrowed until the next
	// decode) until the next I/P picture arrives; flush() renders the last one
	this.displayOrder = !!(options.decodeBPictures && options.displayOrder);
	// extension: with exportMacroblocks, macroblocks() gives the macroblock types and motion vectors of the picture the
	// last decode() rendered (motion detection, overlays) without walking the picture a second time
	this.exportMacroblocks = !!options.exportMacroblocks;
	if (this.exportMacroblocks) { native.setExportMacroblocks(this.decoder, 1); }
	// extension: with concealErrors, each macroblock a damaged picture lacks gets the co-located samples of the picture
	// it predicts from, instead of keeping what the plane held two pictures ago
	this.concealErrors = !!options.concealErrors;
	if (this.concealErrors) { native.setConceal(this.decoder, 1); }
	this.held = null;
	this.decodeFirstFrame = options.decodeFirstFrame !== false;
	this.hasSequenceHeader = false;
};

MPEG1B200.prototype = Object.create(JSMpeg.Decoder.Base.prototype);
MPEG1B200.prototype.constructor = MPEG1B200;

MPEG1B200.prototype.destroy = function() { native.destroy(this.decoder); };
MPEG1B200.prototype.bufferGetIndex = function() { return native.getIndex(this.decoder); };
MPEG1B200.prototype.bufferSetIndex = function(index) { native.setIndex(this.decoder, index); };

MPEG1B200.prototype.bufferWrite = function(buffers) {
	var total = 0;
	for (var i = 0; i < buffers.length; i++) {
		total += native.write(this.decoder, buffers[i]);
	}
	return total;
};

MPEG1B200.prototype.write = function(pts, buffers) {
	JSMpeg.Decoder.Base.prototype.write.call(this, pts, buffers);
	if (!this.hasSequenceHeader && native.hasSequenceHeader(this.decoder)) {
		this.hasSequenceHeader = true;
		this.frameRate = native.getFrameRate(this.decoder);
		this.codedSize = native.getCodedSize(this.decoder);
		this.width = native.getWidth(this.decoder);
		this.height = native.getHeight(this.decoder);
		if (this.destination) {
			this.destination.resize(this.width, this.height);
		}
		if (this.decodeFirstFrame) {
			this.decode();
		}
	}
};

MPEG1B200.prototype.decode = function() {
	var startTime = JSMpeg.Now();
	if (!native.decode(this.decoder)) {
		return false;
	}
	if (this.destination) {
		var p = native.planes(this.decoder);
		this.currentY = p.y; this.currentCr = p.cr; this.currentCb = p.cb;
		var type = this.displayOrder ? native.lastPictureType(this.decoder) : 3;
		if (type === 3) {
			this.destination.render(p.y, p.cr, p.cb, false);
		}
		else if (type === 1 || type === 2) {
			this.flush();
			this.held = {y: p.y.slice(), cr: p.cr.slice(), cb: p.cb.slice()};
		}
	}
	this.advanceDecodedTime(1/this.frameRate);
	if (this.onDecodeCallback) {
		this.onDecodeCallback(this, JSMpeg.Now() - startTime);
	}
	return true;
};

// Uint8Array of 16 bytes per macroblock in raster order (include/jsmpeg_b200.h: jsmpeg_b200_macroblock_t), borrowed
// until the next decode(); null without exportMacroblocks or before the sequence header
MPEG1B200.prototype.macroblocks = function() {
	return this.exportMacroblocks ? (native.macroblocks(this.decoder) || null) : null;
};

MPEG1B200.prototype.flush = function() {
	if (this.held && this.destination) {
		this.destination.render(this.held.y, this.held.cr, this.held.cb, false);
	}
	this.held = null;
};

return MPEG1B200;

})();
